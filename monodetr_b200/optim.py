"""Optimizer of the training step (SURVEY.md 8f-2): the reference's AdamW (lib/helpers/optimizer_helper.py:30-129) as ONE
fused kernel over flat buffers, and `build_optimizer` with the reference's signature / grouping rule (:7-27).

Layout.  The parameters the step updates are the gradient-receiving tensors of `FlatGradBucket` (monodetr_b200.ddp), in the
bucket's order: weight-decay tensors first, then every tensor with 'bias' in its name (weight_decay 0 -- the reference's
rule, :9-16).  At construction the optimizer moves those parameters INTO one flat fp32 buffer (`p.data` becomes a view of
it; values, names, shapes and state_dict are unchanged), keeps exp_avg / exp_avg_sq as two more flat buffers, and takes the
bucket's flat gradient buffer as `g`.  `step()` is then a single HBM-bound launch (`mdb_adamw_step_f32`, 28 bytes per
parameter) instead of ~10 elementwise kernels per tensor; with `device_step=True` the bias-correction factor is computed
on the device by a second, single-thread launch (`mdb_adamw_advance`) from a small device block that also holds the learning
rate, so the whole step can live inside a CUDA graph and a learning-rate schedule still reaches every replay (`sync_hyper`).
`state_dict()` / `load_state_dict()` speak the reference optimizer's checkpoint format.

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
        self.device_step = device_step
        self._count = 0
        # the reference optimizer's parameter numbering (optimizer_helper.py:7-16): every named parameter, biases first
        named = list(model.named_parameters())
        self._ref_groups = [[p for n, p in named if "bias" in n], [p for n, p in named if "bias" not in n]]
        if device_step:
            # MdbAdamwHyper (include/monodetr_b200.h): t, lr, beta1, beta2 as doubles, then step_size as a float
            self._hyper = torch.zeros(5, dtype=torch.float64, device=b.flat.device)
            self._step_size = self._hyper.view(torch.float32)[8:9]
            on_gpu = b.flat.device.type == "cuda"
            self._lr_host = torch.zeros(1, dtype=torch.float64, pin_memory=on_gpu)
            self._lr_uploaded, self._lr_event = None, (torch.cuda.Event() if on_gpu else None)
            self._hyper[2:4] = torch.tensor(betas, dtype=torch.float64)
            self.sync_hyper()

    @property
    def step_count(self):
        """Steps taken so far.  With `device_step=True` the count lives on the device (replays of a captured graph advance it
        without the host), so reading it synchronises; a trainer reads it when it writes a checkpoint, not per step."""
        return int(self._hyper[0].item()) if self.device_step else self._count

    @step_count.setter
    def step_count(self, value):
        if self.device_step:
            self._hyper[0:1].fill_(float(int(value)))
        else:
            self._count = int(value)

    def _lr(self):
        lrs = {g["lr"] for g in self.param_groups}
        if len(lrs) != 1:                              # one flat update, one learning rate (the reference builds both groups alike)
            raise ValueError("FusedAdamW: the parameter groups must share one learning rate, got %s" % sorted(lrs))
        return float(next(iter(lrs)))

    def sync_hyper(self):
        """`device_step=True`: send `param_groups[...]['lr']` to the device block if it differs from the value last sent -- one
        asynchronous 8-byte copy from a pinned word, ordered on the current stream and never part of a captured graph.  `step()`
        calls it when it runs eagerly; a loop that replays a captured step calls it after every scheduler step."""
        if not self.device_step:
            return
        lr = self._lr()
        if lr == self._lr_uploaded:
            return
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("FusedAdamW: the learning rate changed inside a CUDA graph capture; call sync_hyper() before capturing")
        if self._lr_event is not None:
            self._lr_event.synchronize()               # the previous upload has read the pinned word (it was issued an epoch ago)
        self._lr_host[0] = lr
        self._hyper[1:2].copy_(self._lr_host, non_blocking=True)
        if self._lr_event is not None:
            self._lr_event.record()
        self._lr_uploaded = lr

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
        g0 = self.param_groups[-1]                    # betas / eps are kept equal across the two groups (as the reference builds them)
        (beta1, beta2), eps = g0["betas"], g0["eps"]
        wd = max(g["weight_decay"] for g in self.param_groups)
        step_dev = None
        if self.device_step:                          # graph-safe: t, lr and the bias corrections live on the device
            self.sync_hyper()                         # no-op unless a scheduler wrote a new lr (an error inside a capture)
            _lib.call("mdb_adamw_advance", self._hyper)
            step_size, step_dev = 0.0, self._step_size
        else:
            self._count += 1
            step_size = self._lr() * math.sqrt(1 - beta2 ** self._count) / (1 - beta1 ** self._count)
        _lib.call("mdb_adamw_step_f32", self.flat_p, b.flat, self.exp_avg, self.exp_avg_sq, b.numel, b.n_decay, beta1, 1 - beta1, beta2,
                  1 - beta2, eps, wd, step_size, step_dev)
        return loss

    # ---- checkpoints in the reference's format ---------------------------------------------------------------------------------
    def _ref_index(self):
        """id(parameter) -> its index in the packed state_dict of the reference's optimizer."""
        return {id(p): i for i, p in enumerate(self._ref_groups[0] + self._ref_groups[1])}

    def _own_group(self, is_bias):
        """This optimizer's group behind the reference's bias / weight group (a model without biases has the weight group only)."""
        return self.param_groups[0] if is_bias and len(self.param_groups) > 1 else self.param_groups[-1]

    def state_dict(self):
        """What `lib/helpers/optimizer_helper.build_optimizer(cfg, model).state_dict()` holds after the same steps: torch's packed
        form over ALL named parameters, biases (weight_decay 0) then weights; `state[i] = {'step', 'exp_avg', 'exp_avg_sq'}`
        (copies, in the parameter's shape) for the parameters that receive gradients, nothing for the others, and nothing at
        all before the first step.  With `device_step=True` this reads the step count from the device (one synchronisation)."""
        index, b, step = self._ref_index(), self.bucket, self.step_count
        state = {}
        if step > 0:
            for off, p in zip(b.offsets, b.params):
                n = p.numel()
                state[index[id(p)]] = {"step": step, "exp_avg": self.exp_avg[off:off + n].view_as(p).clone(),
                                       "exp_avg_sq": self.exp_avg_sq[off:off + n].view_as(p).clone()}
        state = {i: state[i] for i in sorted(state)}
        groups, start = [], 0
        for is_bias, params in ((True, self._ref_groups[0]), (False, self._ref_groups[1])):
            g = {k: v for k, v in self._own_group(is_bias).items() if k != "params"}
            if is_bias:
                g["weight_decay"] = 0
            g["params"] = list(range(start, start + len(params)))
            start += len(params)
            groups.append(g)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict):
        """Accepts the dict `state_dict()` returns or one saved by the reference's `AdamW` over the same model: the moments are
        scattered into the flat buffers, the hyper-parameters (lr included, as torch does) are taken from the loaded groups, keys
        this class does not know are kept in `param_groups` and otherwise ignored.  All parameters are updated by one kernel with
        ONE step count, so a state whose `step` values differ between parameters, or that holds moments for only some of the
        gradient-receiving parameters, raises ValueError."""
        groups = state_dict["param_groups"]
        if len(groups) != 2 or [len(g["params"]) for g in groups] != [len(g) for g in self._ref_groups]:
            raise ValueError("FusedAdamW.load_state_dict: expected the reference's two groups (biases, weights) over this model's "
                             "%d + %d parameters" % tuple(len(g) for g in self._ref_groups))
        order = list(groups[0]["params"]) + list(groups[1]["params"])
        by_param = {id(p): i for p, i in zip(self._ref_groups[0] + self._ref_groups[1], order)}
        state, b = state_dict["state"], self.bucket
        have = [by_param[id(p)] in state for p in b.params]
        extra = set(state) - {by_param[id(p)] for p in b.params}
        if extra:
            raise ValueError("FusedAdamW.load_state_dict: state for parameters that receive no gradient here: %s" % sorted(extra))
        if any(have) and not all(have):
            raise ValueError("FusedAdamW.load_state_dict: moments are missing for some gradient-receiving parameters")
        steps = {int(state[by_param[id(p)]]["step"]) for p in b.params} if all(have) else {0}
        if len(steps) != 1:
            raise ValueError("FusedAdamW.load_state_dict: one step count for all parameters is required, got %s" % sorted(steps))
        with torch.no_grad():
            self.exp_avg.zero_()
            self.exp_avg_sq.zero_()
            if all(have):
                for off, p in zip(b.offsets, b.params):
                    s, n = state[by_param[id(p)]], p.numel()
                    self.exp_avg[off:off + n].view_as(p).copy_(s["exp_avg"])
                    self.exp_avg_sq[off:off + n].view_as(p).copy_(s["exp_avg_sq"])
        for is_bias in (True, False):
            self._own_group(is_bias).update({k: v for k, v in groups[0 if is_bias else 1].items() if k != "params"})
        self.step_count = steps.pop()
        if self.device_step:
            self._hyper[2:4] = torch.tensor(self.param_groups[-1]["betas"], dtype=torch.float64)
            self.sync_hyper()

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


class CosineWarmupLR(torch.optim.lr_scheduler._LRScheduler):
    """lib/helpers/scheduler_helper.py:68-77: from `init_lr` to the base lr over `num_epoch` epochs along half a cosine."""

    def __init__(self, optimizer, num_epoch, init_lr=0.0, last_epoch=-1):
        self.num_epoch = num_epoch
        self.init_lr = init_lr
        super().__init__(optimizer, last_epoch)

    def get_lr(self):
        return [self.init_lr + (base_lr - self.init_lr) * (1 - math.cos(math.pi * self.last_epoch / self.num_epoch)) / 2
                for base_lr in self.base_lrs]


def build_lr_scheduler(cfg, optimizer, last_epoch):
    """lib/helpers/scheduler_helper.py:6-18: `LambdaLR` multiplying by `decay_rate` at every epoch of `decay_list`, and, with
    `cfg['warmup']`, the 5-epoch cosine warm-up from 1e-5.  Returns (lr_scheduler, warmup_lr_scheduler or None)."""
    def lr_lbmd(cur_epoch):
        cur_decay = 1
        for decay_step in cfg["decay_list"]:
            if cur_epoch >= decay_step:
                cur_decay = cur_decay * cfg["decay_rate"]
        return cur_decay

    lr_scheduler = torch.optim.lr_scheduler.LambdaLR(optimizer, lr_lbmd, last_epoch=last_epoch)
    warmup_lr_scheduler = CosineWarmupLR(optimizer, num_epoch=5, init_lr=0.00001) if cfg["warmup"] else None
    return lr_scheduler, warmup_lr_scheduler
