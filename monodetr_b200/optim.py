"""Optimizers of the training step (SURVEY.md 8f-2): the reference's three `optimizer.type` values (lib/helpers/optimizer_helper.py:
7-27) -- its own AdamW (:30-129), `torch.optim.SGD(momentum=0.9)` and `torch.optim.Adam` -- each as ONE fused kernel over flat
buffers, and `build_optimizer` with the reference's signature / grouping rule.

Layout.  The parameters the step updates are the gradient-receiving tensors of `FlatGradBucket` (monodetr_b200.ddp), in the
bucket's order: weight-decay tensors first, then every tensor with 'bias' in its name (weight_decay 0 -- the reference's
rule, :9-16).  At construction the optimizer moves those parameters INTO one flat fp32 buffer (`p.data` becomes a view of
it; values, names, shapes and state_dict are unchanged), keeps its state (exp_avg / exp_avg_sq, or the momentum buffer) as more
flat buffers, and takes the bucket's flat gradient buffer as `g`.  `step()` is then a single HBM-bound launch
(`mdb_adamw_step_f32` / `mdb_adam_step_f32`, 28 bytes per parameter; `mdb_sgd_step_f32`, 20) instead of several elementwise
kernels per tensor; with `device_step=True` the step count and the step scalars are computed on the device by a second,
single-thread launch (`mdb_*_advance`) from a small device block that also holds the learning rate, so the whole step can live
inside a CUDA graph and a learning-rate schedule still reaches every replay (`sync_hyper`).  `state_dict()` / `load_state_dict()`
speak the reference optimizer's checkpoint format (torch's packed form).

Parameters that never receive a gradient (SURVEY.md appendix C.2: sa_v_proj, query_scale, ref_point_head, label_enc; with
use_dab sa_v_proj, query_scale_bbox, label_enc) are not in the bucket and are left untouched, exactly as the reference's `if p.grad is None: continue` (:95-96) leaves them.
"""
import math

import torch

from . import _lib
from .ddp import FlatGradBucket


class _FlatOptimizer(torch.optim.Optimizer):
    """What the three fused optimizers share: the parameters moved into one flat buffer in bucket order, state buffers of the
    bucket's size, the reference's two groups (biases with weight_decay 0, then weights) in `param_groups`, one learning rate
    for both, the step count (on the device with `device_step=True`, in a block whose first two doubles are t and lr),
    `sync_hyper()` and checkpoints in torch's packed format over all named parameters.  A subclass names its state buffers
    (`STATE`), the size of its device block in doubles (`HYPER_DOUBLES`) and implements `_launch()` and the per-parameter state
    of its checkpoints."""

    STATE = ()
    HYPER_DOUBLES = 2

    def __init__(self, model, bucket, defaults, weight_decay, device_step):
        self.bucket = bucket if bucket is not None else FlatGradBucket(model)
        b = self.bucket
        name = type(self).__name__
        if not b.params[0].is_cuda:
            raise RuntimeError("%s: CUDA parameters required (there is no CPU path)" % name)
        nd = next(i for i, n in enumerate(b.names + ["bias"]) if "bias" in n)          # first no-decay tensor
        groups = [{"params": b.params[nd:], "weight_decay": 0}, {"params": b.params[:nd], "weight_decay": weight_decay}]
        super().__init__([g for g in groups if g["params"]], defaults)
        # parameters -> views of one flat buffer, in bucket order
        self.flat_p = torch.zeros_like(b.flat)
        with torch.no_grad():
            for off, p in zip(b.offsets, b.params):          # 128-byte aligned offsets: vector loads / TMA on parameters keep working
                v = self.flat_p[off:off + p.numel()].view_as(p)
                v.copy_(p)
                p.data = v
        for s in self.STATE:
            setattr(self, s, torch.zeros_like(b.flat))
        self.device_step = device_step
        self._count = 0
        # the reference optimizer's parameter numbering (optimizer_helper.py:7-16): every named parameter, biases first
        named = list(model.named_parameters())
        self._ref_groups = [[p for n, p in named if "bias" in n], [p for n, p in named if "bias" not in n]]
        if device_step:
            self._hyper = torch.zeros(self.HYPER_DOUBLES, dtype=torch.float64, device=b.flat.device)
            on_gpu = b.flat.device.type == "cuda"
            self._lr_host = torch.zeros(1, dtype=torch.float64, pin_memory=on_gpu)
            self._lr_uploaded, self._lr_event = None, (torch.cuda.Event() if on_gpu else None)

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
            raise ValueError("%s: the parameter groups must share one learning rate, got %s" % (type(self).__name__, sorted(lrs)))
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
            raise RuntimeError("%s: the learning rate changed inside a CUDA graph capture; call sync_hyper() before capturing"
                               % type(self).__name__)
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
        self._grads_in_bucket()
        if self.device_step:
            self.sync_hyper()                         # no-op unless a scheduler wrote a new lr (an error inside a capture)
        self._launch(max(g["weight_decay"] for g in self.param_groups))
        return loss

    # ---- checkpoints in torch's packed format ------------------------------------------------------------------------------------
    def _ref_index(self):
        """id(parameter) -> its index in the packed state_dict of the reference's optimizer."""
        return {id(p): i for i, p in enumerate(self._ref_groups[0] + self._ref_groups[1])}

    def _own_group(self, is_bias):
        """This optimizer's group behind the reference's bias / weight group (a model without biases has the weight group only)."""
        return self.param_groups[0] if is_bias and len(self.param_groups) > 1 else self.param_groups[-1]

    def _views(self, off, p):
        """(name, view in the parameter's shape) of every state buffer at one parameter."""
        return [(s, getattr(self, s)[off:off + p.numel()].view_as(p)) for s in self.STATE]

    def _param_state(self, views, step):
        return {"step": step, **{s: v.clone() for s, v in views}}

    def state_dict(self):
        """What the reference's `build_optimizer(cfg, model).state_dict()` holds after the same steps: torch's packed form over ALL
        named parameters, biases (weight_decay 0) then weights; per-parameter state (copies, in the parameter's shape) for the
        parameters that receive gradients, nothing for the others, and nothing at all before the first step.  With
        `device_step=True` this reads the step count from the device (one synchronisation)."""
        index, b, step = self._ref_index(), self.bucket, self.step_count
        state = {}
        if step > 0:
            for off, p in zip(b.offsets, b.params):
                state[index[id(p)]] = self._param_state(self._views(off, p), step)
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

    def _check_groups(self, groups):
        """Refuses loaded hyper-parameters the flat step does not implement."""

    def _loaded_step(self, states):
        """The one step count of a complete loaded state (`states`: one dict per gradient-receiving parameter)."""
        steps = {int(s["step"]) for s in states}
        if len(steps) != 1:
            raise ValueError("%s.load_state_dict: one step count for all parameters is required, got %s"
                             % (type(self).__name__, sorted(steps)))
        return steps.pop()

    def _after_load(self):
        pass

    def load_state_dict(self, state_dict):
        """Accepts the dict `state_dict()` returns or one saved by the reference's optimizer of the same type over the same model:
        the state is scattered into the flat buffers, the hyper-parameters (lr included, as torch does) are taken from the loaded
        groups, keys this class does not know are kept in `param_groups` and otherwise ignored.  All parameters are updated by one
        kernel with ONE step count, so a state whose `step` values differ between parameters, or that holds state for only some
        of the gradient-receiving parameters, raises ValueError."""
        name = type(self).__name__
        groups = state_dict["param_groups"]
        if len(groups) != 2 or [len(g["params"]) for g in groups] != [len(g) for g in self._ref_groups]:
            raise ValueError("%s.load_state_dict: expected the reference's two groups (biases, weights) over this model's "
                             "%d + %d parameters" % ((name,) + tuple(len(g) for g in self._ref_groups)))
        self._check_groups(groups)
        order = list(groups[0]["params"]) + list(groups[1]["params"])
        by_param = {id(p): i for p, i in zip(self._ref_groups[0] + self._ref_groups[1], order)}
        state, b = state_dict["state"], self.bucket
        have = [by_param[id(p)] in state for p in b.params]
        extra = set(state) - {by_param[id(p)] for p in b.params}
        if extra:
            raise ValueError("%s.load_state_dict: state for parameters that receive no gradient here: %s" % (name, sorted(extra)))
        if any(have) and not all(have):
            raise ValueError("%s.load_state_dict: moments are missing for some gradient-receiving parameters" % name)
        step = self._loaded_step([state[by_param[id(p)]] for p in b.params]) if all(have) else 0
        with torch.no_grad():
            for s in self.STATE:
                getattr(self, s).zero_()
            if all(have):
                for off, p in zip(b.offsets, b.params):
                    loaded = state[by_param[id(p)]]
                    for s, v in self._views(off, p):
                        v.copy_(loaded[s])
        for is_bias in (True, False):
            self._own_group(is_bias).update({k: v for k, v in groups[0 if is_bias else 1].items() if k != "params"})
        self.step_count = step
        self._after_load()
        if self.device_step:
            self.sync_hyper()

    def zero_grad(self, set_to_none=True):
        self.bucket.zero()


class FusedAdamW(_FlatOptimizer):
    """Same constructor arguments, `param_groups` keys and update rule as the reference's AdamW; amsgrad is not supported."""

    STATE = ("exp_avg", "exp_avg_sq")
    HYPER_DOUBLES = 5

    def __init__(self, model, bucket: FlatGradBucket = None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, device_step=False):
        if lr < 0.0 or eps < 0.0 or not (0.0 <= betas[0] < 1.0) or not (0.0 <= betas[1] < 1.0):
            raise ValueError("invalid AdamW hyper-parameters")
        super().__init__(model, bucket, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False), weight_decay,
                         device_step)
        if device_step:
            # MdbAdamwHyper (include/monodetr_b200.h): t, lr, beta1, beta2 as doubles, then step_size as a float
            self._step_size = self._hyper.view(torch.float32)[8:9]
            self._after_load()
            self.sync_hyper()

    def _launch(self, wd):
        b = self.bucket
        g0 = self.param_groups[-1]                    # betas / eps are kept equal across the two groups (as the reference builds them)
        (beta1, beta2), eps = g0["betas"], g0["eps"]
        step_dev = None
        if self.device_step:                          # graph-safe: t, lr and the bias corrections live on the device
            _lib.call("mdb_adamw_advance", self._hyper)
            step_size, step_dev = 0.0, self._step_size
        else:
            self._count += 1
            step_size = self._lr() * math.sqrt(1 - beta2 ** self._count) / (1 - beta1 ** self._count)
        _lib.call("mdb_adamw_step_f32", self.flat_p, b.flat, self.exp_avg, self.exp_avg_sq, b.numel, b.n_decay, beta1, 1 - beta1, beta2,
                  1 - beta2, eps, wd, step_size, step_dev)

    def _after_load(self):
        if self.device_step:
            self._hyper[2:4] = torch.tensor(self.param_groups[-1]["betas"], dtype=torch.float64)


class FusedSGD(_FlatOptimizer):
    """The reference's `sgd`: `torch.optim.SGD(groups, lr, momentum=0.9)` (dampening 0, no Nesterov, no `maximize`) as one launch
    over the flat buffers (`mdb_sgd_step_f32`, 20 bytes per parameter), with torch's `param_groups` keys and checkpoint format
    (`state[i] = {'momentum_buffer'}`).  torch creates the momentum buffers on the first step (buf = d) and accumulates into
    them afterwards; here that choice is made by the kernel, from the device block's step count with `device_step=True`, so a
    captured step is right whether or not the buffers exist.  A state loaded with momentum buffers counts as one step taken
    (torch's SGD keeps no step count); `step_count` counts from there."""

    STATE = ("momentum_buffer",)
    HYPER_DOUBLES = 2

    def __init__(self, model, bucket: FlatGradBucket = None, lr=1e-3, momentum=0.9, weight_decay=0, device_step=False):
        if lr < 0.0 or not momentum > 0.0 or weight_decay < 0.0:
            raise ValueError("invalid SGD hyper-parameters (the fused step needs momentum > 0)")
        super().__init__(model, bucket, dict(lr=lr, momentum=momentum, dampening=0, nesterov=False, maximize=False, foreach=None,
                                             differentiable=False, fused=None), weight_decay, device_step)
        if device_step:
            self.sync_hyper()                         # MdbSgdHyper (include/monodetr_b200.h): t, lr as doubles

    def _launch(self, wd):
        b = self.bucket
        momentum = self.param_groups[-1]["momentum"]
        if self.device_step:
            _lib.call("mdb_sgd_advance", self._hyper)
            lr, first, hyper = 0.0, 0, self._hyper
        else:
            self._count += 1
            lr, first, hyper = self._lr(), int(self._count == 1), None
        _lib.call("mdb_sgd_step_f32", self.flat_p, b.flat, self.momentum_buffer, b.numel, b.n_decay, momentum, wd, lr, first, hyper)

    def _param_state(self, views, step):
        return {s: v.clone() for s, v in views}

    def _loaded_step(self, states):
        return 1

    def _check_groups(self, groups):
        for g in groups:
            if g.get("dampening", 0) != 0 or g.get("nesterov", False) or g.get("maximize", False) or not g.get("momentum", 0) > 0:
                raise ValueError("FusedSGD.load_state_dict: dampening, nesterov, maximize and momentum 0 are not supported")


class FusedAdam(_FlatOptimizer):
    """The reference's `adam`: `torch.optim.Adam(groups, lr)` (L2 weight decay added to the gradient; no amsgrad, `maximize` or
    decoupled decay) as one launch over the flat buffers (`mdb_adam_step_f32`, 28 bytes per parameter), with torch's
    `param_groups` keys and checkpoint format (`state[i] = {'step': float32 tensor, 'exp_avg', 'exp_avg_sq'}`).  The two step
    scalars, lr / (1 - beta1^t) and sqrt(1 - beta2^t), are fp64 host values in eager mode and come from the device block with
    `device_step=True` (`mdb_adam_advance`)."""

    STATE = ("exp_avg", "exp_avg_sq")
    HYPER_DOUBLES = 5

    def __init__(self, model, bucket: FlatGradBucket = None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, device_step=False):
        if lr < 0.0 or eps < 0.0 or not (0.0 <= betas[0] < 1.0) or not (0.0 <= betas[1] < 1.0) or weight_decay < 0.0:
            raise ValueError("invalid Adam hyper-parameters")
        super().__init__(model, bucket, dict(lr=lr, betas=betas, eps=eps, amsgrad=False, maximize=False, foreach=None,
                                             capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False),
                         weight_decay, device_step)
        if device_step:
            # MdbAdamHyper (include/monodetr_b200.h): t, lr, beta1, beta2 as doubles, then neg_step and bc2_sqrt as floats
            self._scalars = self._hyper.view(torch.float32)[8:10]
            self._after_load()
            self.sync_hyper()

    def _launch(self, wd):
        b = self.bucket
        g0 = self.param_groups[-1]
        (beta1, beta2), eps = g0["betas"], g0["eps"]
        if self.device_step:
            _lib.call("mdb_adam_advance", self._hyper)
            neg_step, bc2_sqrt, hyper = 0.0, 1.0, self._hyper
        else:                                         # torch/optim/adam.py, capturable=False: Python floats
            self._count += 1
            t = float(self._count)
            bc1, bc2 = 1 - beta1 ** t, 1 - beta2 ** t
            neg_step, bc2_sqrt, hyper = (self._lr() / bc1) * -1, bc2 ** 0.5, None
        _lib.call("mdb_adam_step_f32", self.flat_p, b.flat, self.exp_avg, self.exp_avg_sq, b.numel, b.n_decay, 1 - beta1, beta2,
                  1 - beta2, eps, wd, neg_step, bc2_sqrt, hyper)

    def _param_state(self, views, step):
        return {"step": torch.tensor(float(step), dtype=torch.float32), **{s: v.clone() for s, v in views}}

    def _check_groups(self, groups):
        for g in groups:
            if g.get("amsgrad", False) or g.get("maximize", False) or g.get("decoupled_weight_decay", False):
                raise ValueError("FusedAdam.load_state_dict: amsgrad, maximize and decoupled_weight_decay are not supported")

    def _after_load(self):
        if self.device_step:
            self._hyper[2:4] = torch.tensor(self.param_groups[-1]["betas"], dtype=torch.float64)


def build_optimizer(cfg_optimizer, model, bucket=None):
    """lib/helpers/optimizer_helper.py:7-27: `adamw`, `sgd` (momentum 0.9) and `adam` (torch's defaults otherwise), each served by
    its fused kernel over the reference's 'bias'-in-name grouping.  Built eagerly (`device_step=False`); a loop that replays a
    captured step constructs the class itself with `device_step=True`."""
    kind, lr, wd = cfg_optimizer["type"], cfg_optimizer["lr"], cfg_optimizer["weight_decay"]
    if kind == "adamw":
        return FusedAdamW(model, bucket, lr=lr, weight_decay=wd)
    if kind == "sgd":
        return FusedSGD(model, bucket, lr=lr, momentum=0.9, weight_decay=wd)
    if kind == "adam":
        return FusedAdam(model, bucket, lr=lr, weight_decay=wd)
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
