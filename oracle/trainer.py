"""The reference training loop's control flow (lib/helpers/trainer_helper.py:44-114 with scheduler_helper.py:6-18, 68-77 and
save_helper.py) restated in plain Python, without torch: which learning rate every epoch trains with, which log lines appear, which
checkpoint files exist afterwards and what they record.  Pinned to the reference itself by tests/test_oracle_trainer.py.

Both schedulers write the one optimizer's lr: `LambdaLR` is constructed first (lr = base * decay(0)), the warm-up second
(lr = init_lr), so training starts at init_lr.  After epoch e the warm-up steps while e < 5, afterwards `LambdaLR` does -- and its
epoch counter only starts then, so the decay epochs are counted from the end of the warm-up.  On resume the lr of the first epoch
is the one saved in the checkpoint, `LambdaLR.last_epoch` is set to epoch - 1 and the warm-up starts over from its first step."""
import math

WARMUP_EPOCHS, WARMUP_INIT_LR = 5, 0.00001


def decay(sched_cfg, epoch):
    d = 1
    for step in sched_cfg["decay_list"]:
        if epoch >= step:
            d = d * sched_cfg["decay_rate"]
    return d


def warmup_lr(base_lr, k):
    return WARMUP_INIT_LR + (base_lr - WARMUP_INIT_LR) * (1 - math.cos(math.pi * k / WARMUP_EPOCHS)) / 2


def simulate(cfg, sched_cfg, base_lr, ap_script=None, resume=None):
    """`resume`: None or the (epoch, best_result, best_epoch, lr) of the checkpoint to continue from.  Returns the lr of every
    epoch trained, the logger lines and {file name: [epoch, best_result, best_epoch]} of the files written."""
    lambda_epoch, warm_epoch = 0, 0
    lr = warmup_lr(base_lr, 0) if sched_cfg["warmup"] else base_lr * decay(sched_cfg, 0)
    epoch, best_result, best_epoch, lines = 0, 0, 0, []
    if resume is not None:
        epoch, best_result, best_epoch, lr = resume
        lambda_epoch = epoch - 1
        lines += ["Loading Checkpoint... Best Result:{}, Best Epoch:{}".format(best_result, best_epoch)]
    lrs, files, tests = [], {}, 0
    for e in range(epoch, cfg["max_epoch"]):
        lrs.append(lr)
        epoch += 1
        if sched_cfg["warmup"] and e < WARMUP_EPOCHS:
            warm_epoch += 1
            lr = warmup_lr(base_lr, warm_epoch)
        else:
            lambda_epoch += 1
            lr = base_lr * decay(sched_cfg, lambda_epoch)
        if epoch % cfg["save_frequency"] == 0:
            files[("checkpoint_epoch_%d" % epoch if cfg["save_all"] else "checkpoint") + ".pth"] = [epoch, best_result, best_epoch]
            if ap_script is not None:
                lines.append("Test Epoch {}".format(epoch))
                cur = ap_script[tests]
                tests += 1
                if cur > best_result:
                    best_result, best_epoch = cur, epoch
                    files["checkpoint_best.pth"] = [epoch, best_result, best_epoch]
                lines.append("Best Result:{}, epoch:{}".format(best_result, best_epoch))
    lines.append("Best Result:{}, epoch:{}".format(best_result, best_epoch))
    return {"lrs": lrs, "logger": lines, "files": files}
