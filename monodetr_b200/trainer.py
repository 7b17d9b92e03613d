"""Drop-in for the reference's lib/helpers/trainer_helper.py `Trainer`: same constructor, `train()`, `train_one_epoch(epoch)`,
`prepare_targets(targets, batch_size)`, attributes (`tester`, `epoch`, `best_result`, `best_epoch`, `output_dir`), control flow,
printed text, log lines and checkpoint files (`checkpoint.pth`, `checkpoint_epoch_N.pth`, `checkpoint_best.pth` with the keys
`epoch, model_state, optimizer_state, best_result, best_epoch`), so either code base resumes from the other's files.

Two ways to run an iteration:

* Graph path -- `loss` is this package's device `SetCriterion`, `optimizer` one of the fused optimizers of `optim`
  (`FusedAdamW`, `FusedSGD`, `FusedAdam`) built with `device_step=True`, and the environment variable MDB_NO_GRAPH is unset.  The
  batch is copied into static device buffers and `zero grads, forward, criterion, weighted sum, backward, optimizer step, loss
  log` is replayed as ONE CUDA graph.  The first batch of a shape runs eagerly (it warms the lazily
  built state and is an ordinary training step), the second is captured -- capturing executes nothing -- and replayed, so every
  batch trains exactly once and the parameters follow the eager loop's trajectory.  One graph per batch shape, at most
  `MAX_GRAPHS` (the loader's short last batch is the second); further shapes run eagerly.  The loss terms are logged on the device
  (`criterion.LossLog`): the block printed every 30 batches appears as soon as its copy has arrived, at the latest at the end of
  the epoch, and no step waits for the host.  The learning rate reaches the replayed step through `optimizer.sync_hyper()`.
  With torch.distributed initialised the captured region ends after backward; the gradient all-reduce and the optimizer's two
  launches follow it, parameters are broadcast from rank 0 at construction and only rank 0 prints, logs and saves.  With
  this package's `Tester` attached, every rank runs its `inference()` / `evaluate()` (it splits the pass over the ranks) and
  so keeps the same `best_result` / `best_epoch`; any other tester runs on rank 0 alone.
* Eager path -- anything else (the reference's own criterion, a torch optimizer): the reference's loop as it is written, with
  `prepare_targets` and the `.item()` log.

The dropout seed (`kernels.master_seed`) is not part of the reference's checkpoint format and is not saved.
"""
import os

import numpy as np
import torch
import torch.distributed as dist

try:
    import tqdm
except ImportError:                       # progress bars are decoration: without tqdm there are none
    tqdm = None


def get_checkpoint_state(model=None, optimizer=None, epoch=None, best_result=None, best_epoch=None):
    """save_helper.py:13-23"""
    model_state = None
    if model is not None:
        model_state = model.module.state_dict() if isinstance(model, torch.nn.DataParallel) else model.state_dict()
        if isinstance(model, torch.nn.DataParallel):
            model_state = type(model_state)((k, v.cpu()) for k, v in model_state.items())
    return {"epoch": epoch, "model_state": model_state, "optimizer_state": optimizer.state_dict() if optimizer is not None else None,
            "best_result": best_result, "best_epoch": best_epoch}


def save_checkpoint(state, filename):
    torch.save(state, "{}.pth".format(filename))


def load_checkpoint(model, optimizer, filename, map_location, logger=None):
    """save_helper.py:31-46: returns (epoch, best_result, best_epoch)."""
    if not os.path.isfile(filename):
        raise FileNotFoundError(filename)
    logger.info("==> Loading from checkpoint '{}'".format(filename))
    checkpoint = torch.load(filename, map_location=map_location, weights_only=False)
    if model is not None and checkpoint["model_state"] is not None:
        model.load_state_dict(checkpoint["model_state"])
    if optimizer is not None and checkpoint["optimizer_state"] is not None:
        optimizer.load_state_dict(checkpoint["optimizer_state"])
    logger.info("==> Done")
    return checkpoint.get("epoch", -1), checkpoint.get("best_result", 0.0), checkpoint.get("best_epoch", 0.0)


def _world():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def reduce_dict(input_dict):
    """utils/misc.py:135-159: the mean over ranks of every value, keys in sorted order; the dict itself in a single process."""
    world = _world()
    if world < 2:
        return input_dict
    with torch.no_grad():
        names = sorted(input_dict.keys())
        values = torch.stack([input_dict[k] for k in names], dim=0)
        dist.all_reduce(values)
        values /= world
    return dict(zip(names, values))


def print_losses(batch_idx, log):
    """The block of trainer_helper.py:155-167."""
    flags = [True] * 5
    print("----", batch_idx, "----")
    print("%s: %.2f, " % ("loss_detr", log["loss_detr"]))
    for key, val in log.items():
        if key == "loss_detr":
            continue
        if any(d in key for d in "012345"):
            if flags[int(key[-1])]:
                print("")
                flags[int(key[-1])] = False
        print("%s: %.2f, " % (key, val), end="")
    print("")
    print("")


class _Progress:
    def __init__(self, **kw):
        self.bar = tqdm.tqdm(**kw) if tqdm is not None else None

    def update(self):
        if self.bar is not None:
            self.bar.update()

    def close(self):
        if self.bar is not None:
            self.bar.close()


class _CapturedStep:
    """One replayable iteration and the static buffers it reads."""

    def __init__(self, inputs, calibs, img_sizes, tgt):
        self.inputs, self.calibs, self.img_sizes = inputs.clone(), calibs.clone(), img_sizes.clone()
        self.tgt = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in tgt.items()}
        self.graph, self.grads = None, None

    def load(self, inputs, calibs, img_sizes, tgt):
        self.inputs.copy_(inputs, non_blocking=True)
        self.calibs.copy_(calibs, non_blocking=True)
        self.img_sizes.copy_(img_sizes, non_blocking=True)
        for k, v in self.tgt.items():
            if torch.is_tensor(v):
                v.copy_(tgt[k], non_blocking=True)


class Trainer(object):
    MAX_GRAPHS = 2
    PRINT_EVERY = 30

    def __init__(self, cfg, model, optimizer, train_loader, test_loader, lr_scheduler, warmup_lr_scheduler, logger, loss, model_name):
        self.cfg = cfg
        self.model = model
        self.optimizer = optimizer
        self.train_loader = train_loader
        self.test_loader = test_loader
        self.lr_scheduler = lr_scheduler
        self.warmup_lr_scheduler = warmup_lr_scheduler
        self.logger = logger
        self.epoch = 0
        self.best_result = 0
        self.best_epoch = 0
        self.device = torch.device("cuda" if torch.cuda.is_available() else "cpu")
        self.detr_loss = loss
        self.model_name = model_name
        self.output_dir = os.path.join("./" + cfg["save_path"], model_name)
        self.tester = None

        from .criterion import SetCriterion
        from .optim import FusedAdam, FusedAdamW, FusedSGD
        self.graph_path = (isinstance(loss, SetCriterion) and isinstance(optimizer, (FusedAdamW, FusedSGD, FusedAdam)) and optimizer.device_step
                           and not os.environ.get("MDB_NO_GRAPH"))
        self._steps = {}                  # batch shape -> _CapturedStep
        self._seen = {}                   # batch shape -> batches of that shape so far
        self._log = None
        self.is_main = not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0

        # loading pretrain/resume model
        if cfg.get("pretrain_model"):
            assert os.path.exists(cfg["pretrain_model"])
            load_checkpoint(model=self.model, optimizer=None, filename=cfg["pretrain_model"], map_location=self.device, logger=self.logger)

        if cfg.get("resume_model", None):
            resume_model_path = os.path.join(self.output_dir, "checkpoint.pth")
            assert os.path.exists(resume_model_path)
            self.epoch, self.best_result, self.best_epoch = load_checkpoint(
                model=self.model.to(self.device), optimizer=self.optimizer, filename=resume_model_path, map_location=self.device,
                logger=self.logger)
            self.lr_scheduler.last_epoch = self.epoch - 1
            self.logger.info("Loading Checkpoint... Best Result:{}, Best Epoch:{}".format(self.best_result, self.best_epoch))

        if _world() > 1:
            from .ddp import broadcast_parameters
            broadcast_parameters(self.model)

    @property
    def live_graphs(self):
        return sum(1 for s in self._steps.values() if s.graph is not None)

    def _tester_splits(self):
        from .tester import Tester                # tester imports this module
        return isinstance(self.tester, Tester)

    def train(self):
        start_epoch = self.epoch

        progress_bar = _Progress(iterable=range(start_epoch, self.cfg["max_epoch"]), dynamic_ncols=True, leave=True, desc="epochs")
        best_result = self.best_result
        best_epoch = self.best_epoch
        for epoch in range(start_epoch, self.cfg["max_epoch"]):
            # reset random seed
            # ref: https://github.com/pytorch/pytorch/issues/5059
            np.random.seed(np.random.get_state()[1][0] + epoch)
            # train one epoch
            self.train_one_epoch(epoch)
            self.epoch += 1

            # update learning rate
            if self.warmup_lr_scheduler is not None and epoch < 5:
                self.warmup_lr_scheduler.step()
            else:
                self.lr_scheduler.step()
            if hasattr(self.optimizer, "sync_hyper"):
                self.optimizer.sync_hyper()           # the new lr reaches the device block a replayed step reads

            # save trained model; rank 0 saves and logs.  This package's Tester splits its pass over the ranks, so every rank
            # runs it; any other tester (the reference's, which does not split) runs on rank 0 alone, as in the reference
            if (self.epoch % self.cfg["save_frequency"]) == 0:
                if self.is_main:
                    os.makedirs(self.output_dir, exist_ok=True)
                    if self.cfg["save_all"]:
                        ckpt_name = os.path.join(self.output_dir, "checkpoint_epoch_%d" % self.epoch)
                    else:
                        ckpt_name = os.path.join(self.output_dir, "checkpoint")

                    save_checkpoint(get_checkpoint_state(self.model, self.optimizer, self.epoch, best_result, best_epoch), ckpt_name)

                if self.tester is not None and (self.is_main or self._tester_splits()):
                    if self.is_main:
                        self.logger.info("Test Epoch {}".format(self.epoch))
                    self.tester.inference()
                    cur_result = self.tester.evaluate()
                    if cur_result > best_result:
                        best_result = cur_result
                        best_epoch = self.epoch
                        if self.is_main:
                            ckpt_name = os.path.join(self.output_dir, "checkpoint_best")
                            save_checkpoint(get_checkpoint_state(self.model, self.optimizer, self.epoch, best_result, best_epoch), ckpt_name)
                    if self.is_main:
                        self.logger.info("Best Result:{}, epoch:{}".format(best_result, best_epoch))

            progress_bar.update()

        if self.is_main:
            self.logger.info("Best Result:{}, epoch:{}".format(best_result, best_epoch))

        return None

    def train_one_epoch(self, epoch):
        torch.set_grad_enabled(True)
        self.model.train()
        if self.is_main:
            print(">>>>>>> Epoch:", str(epoch) + ":")

        progress_bar = _Progress(total=len(self.train_loader), leave=(self.epoch + 1 == self.cfg["max_epoch"]), desc="iters")
        pending = []                      # graph path: (batch_idx, log record) whose copy may still be in flight
        for batch_idx, (inputs, calibs, targets, info) in enumerate(self.train_loader):
            inputs = inputs.to(self.device)
            calibs = calibs.to(self.device)
            for key in targets.keys():
                targets[key] = targets[key].to(self.device)
            img_sizes = targets["img_size"]
            if self.graph_path:
                self._graph_iteration(inputs, calibs, targets, img_sizes)
                if batch_idx % self.PRINT_EVERY == 0:
                    pending.append((batch_idx, self._log.fetch(self._log.pushed - 1)))
                while pending and pending[0][1].ready():
                    self._print(*pending.pop(0))
            else:
                self._eager_iteration(batch_idx, inputs, calibs, targets, img_sizes)
            progress_bar.update()
        for item in pending:              # the end of the epoch is the one place that waits for the log
            self._print(*item)
        progress_bar.close()

    def _print(self, batch_idx, record):
        log = record.read()
        if self.is_main:
            print_losses(batch_idx, log)

    # ---- the reference's iteration, trainer_helper.py:128-170 ------------------------------------------------------------------
    def _eager_iteration(self, batch_idx, inputs, calibs, targets, img_sizes):
        targets = self.prepare_targets(targets, inputs.shape[0])
        dn_args = None
        if self.cfg["use_dn"]:
            dn_args = (targets, self.cfg["scalar"], self.cfg["label_noise_scale"], self.cfg["box_noise_scale"], self.cfg["num_patterns"])
        # train one batch
        self.optimizer.zero_grad()
        outputs = self.model(inputs, calibs, targets, img_sizes, dn_args=dn_args)
        mask_dict = None
        detr_losses_dict = self.detr_loss(outputs, targets, mask_dict)

        weight_dict = self.detr_loss.weight_dict
        detr_losses_dict_weighted = [detr_losses_dict[k] * weight_dict[k] for k in detr_losses_dict.keys() if k in weight_dict]
        detr_losses = sum(detr_losses_dict_weighted)

        detr_losses_dict = reduce_dict(detr_losses_dict)
        detr_losses_dict_log = {}
        detr_losses_log = 0
        for k in detr_losses_dict.keys():
            if k in weight_dict:
                detr_losses_dict_log[k] = (detr_losses_dict[k] * weight_dict[k]).item()
                detr_losses_log += detr_losses_dict_log[k]
        detr_losses_dict_log["loss_detr"] = detr_losses_log
        self.last_log = detr_losses_dict_log

        if batch_idx % self.PRINT_EVERY == 0 and self.is_main:
            print_losses(batch_idx, detr_losses_dict_log)

        detr_losses.backward()
        self._all_reduce_grads()
        self.optimizer.step()

    def _all_reduce_grads(self):
        world = _world()
        if world < 2:
            return
        bucket = getattr(self.optimizer, "bucket", None)
        if bucket is not None:
            bucket.static_grads = None                # an eager backward: pack from .grad, not from a captured step's tensors
            bucket.all_reduce()
            return
        for p in self.model.parameters():
            if p.grad is not None:
                dist.all_reduce(p.grad)
                p.grad /= world

    # ---- the iteration as a replayed CUDA graph ----------------------------------------------------------------------------------
    def _device_step(self, inputs, calibs, img_sizes, tgt):
        """Everything of one iteration that a graph can hold.  `dn_args` is None: `use_dn` does nothing in the model."""
        self.optimizer.zero_grad()
        outputs = self.model(inputs, calibs, None, img_sizes, dn_args=None)
        self.detr_loss(outputs, tgt)
        if self._log is None:
            from .criterion import LossLog
            self._log = LossLog(self.detr_loss, self.detr_loss._last_losses.shape[0], inputs.device)
        self.detr_loss.weighted_sum().backward()
        if _world() < 2:
            self.optimizer.step()
        self._log.push()

    def _graph_iteration(self, inputs, calibs, targets, img_sizes):
        from .criterion import pack_targets
        tgt = pack_targets(targets, self.device)
        img_sizes = img_sizes.to(self.device)
        key = (tuple(inputs.shape), tuple(tgt["mask"].shape))
        seen = self._seen.get(key, 0)
        self._seen[key] = seen + 1
        step = self._steps.get(key)
        bucket = self.optimizer.bucket
        if step is None and seen >= 1 and self.live_graphs < self.MAX_GRAPHS:
            # second batch of this shape: capture (nothing executes), then replay below -- this batch's one training step
            step = self._steps[key] = _CapturedStep(inputs, calibs, img_sizes, tgt)
            self.optimizer.sync_hyper()
            step.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(step.graph):
                self._device_step(step.inputs, step.calibs, step.img_sizes, step.tgt)
            step.grads = [p.grad if p.grad is not None else torch.zeros_like(v) for p, v in zip(bucket.params, bucket.views)]
        if step is not None:
            step.load(inputs, calibs, img_sizes, tgt)
            step.graph.replay()
            self._log.replayed()
            if _world() > 1:
                bucket.static_grads = step.grads      # the tensors this graph's backward has just rewritten
                bucket.all_reduce()
                self.optimizer.step()
            return
        # first batch of a shape (or more shapes than graphs): an ordinary eager step, on a side stream as a capture warm-up wants it
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._device_step(inputs, calibs, img_sizes, tgt)
            if _world() > 1:
                self._all_reduce_grads()
                self.optimizer.step()
        torch.cuda.current_stream().wait_stream(side)

    def prepare_targets(self, targets, batch_size):
        targets_list = []
        mask = targets["mask_2d"]

        key_list = ["labels", "boxes", "calibs", "depth", "size_3d", "heading_bin", "heading_res", "boxes_3d"]
        for bz in range(batch_size):
            target_dict = {}
            for key, val in targets.items():
                if key in key_list:
                    target_dict[key] = val[bz][mask[bz]]
            targets_list.append(target_dict)
        return targets_list
