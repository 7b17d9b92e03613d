"""Generate tests/golden/trainer.npz by running the UNMODIFIED reference `Trainer` (lib/helpers/trainer_helper.py), its
`build_optimizer` / `AdamW` and its `build_lr_scheduler` on the CPU over the stubs of tests/trainer_stubs.py.  Recorded: the lr of
every step, the printed text, the logger lines, the checkpoint files with their epoch / best_result / best_epoch, the structure of
the optimizer's state_dict, the final parameters -- for a straight run with a tester (A) and for a run resumed from
`checkpoint.pth` (B).  Only data goes into the repository.

    python tools/gen_golden_trainer.py
"""
import contextlib
import io
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]
import ref_shims  # noqa: E402
import trainer_stubs as S  # noqa: E402


def run(trainer_cls, build_optimizer, build_lr_scheduler, cfg, tester=None, model=None):
    """One `Trainer.train()` in the current directory; returns what the fixture records."""
    model = model or S.StubModel()
    optimizer = build_optimizer(S.OPT_CFG, model)
    lr_scheduler, warmup = build_lr_scheduler(S.SCHED_CFG, optimizer, last_epoch=-1)
    logger = S.ListLogger()
    trainer = trainer_cls(cfg=cfg, model=model, optimizer=optimizer, train_loader=S.make_loader(), test_loader=None,
                          lr_scheduler=lr_scheduler, warmup_lr_scheduler=warmup, logger=logger, loss=S.StubCriterion(), model_name="stub")
    trainer.tester = tester
    lrs, step = [], optimizer.step

    def counting_step(*a, **k):
        lrs.append([g["lr"] for g in optimizer.param_groups])
        return step(*a, **k)
    optimizer.step = counting_step
    np.random.seed(7)
    out = io.StringIO()
    with contextlib.redirect_stdout(out), contextlib.redirect_stderr(io.StringIO()):
        trainer.train()
    files = {}
    for f in sorted(os.listdir(trainer.output_dir)):
        c = torch.load(os.path.join(trainer.output_dir, f), weights_only=False)
        files[f] = [c["epoch"], c["best_result"], c["best_epoch"]]
    return {"lrs": lrs, "stdout": out.getvalue(), "logger": logger.lines, "files": files, "optimizer": optimizer, "model": model,
            "numpy_seed": int(np.random.get_state()[1][0])}


def structure(sd):
    return {"state": {str(i): {"step": int(s["step"]), "shapes": {k: list(v.shape) for k, v in s.items() if torch.is_tensor(v)}}
                      for i, s in sd["state"].items()},
            "param_groups": [{k: (list(v) if isinstance(v, (tuple, list)) else v) for k, v in g.items()} for g in sd["param_groups"]]}


def main():
    sys.path.insert(0, ref_shims.REF_ROOT)
    from lib.helpers.optimizer_helper import build_optimizer
    from lib.helpers.scheduler_helper import build_lr_scheduler
    from lib.helpers.trainer_helper import Trainer
    arrays, meta = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        a = run(Trainer, build_optimizer, build_lr_scheduler, dict(S.CFG), tester=S.StubTester())
        meta["A"] = {k: a[k] for k in ("lrs", "stdout", "logger", "files", "numpy_seed")}
        meta["A"]["state_dict"] = structure(a["optimizer"].state_dict())
        for n, p in a["model"].named_parameters():
            arrays["A/" + n] = p.detach().numpy().copy()
        sd = a["optimizer"].state_dict()
        for i, s in sd["state"].items():
            arrays[f"A/exp_avg/{i}"], arrays[f"A/exp_avg_sq/{i}"] = s["exp_avg"].numpy().copy(), s["exp_avg_sq"].numpy().copy()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        cfg = dict(S.CFG, save_all=False, max_epoch=3)
        b1 = run(Trainer, build_optimizer, build_lr_scheduler, cfg)
        b2 = run(Trainer, build_optimizer, build_lr_scheduler, dict(cfg, max_epoch=7, resume_model=True))
        meta["B"] = {"first": {k: b1[k] for k in ("lrs", "logger", "files")}, "resumed": {k: b2[k] for k in ("lrs", "logger", "files")}}
        for n, p in b2["model"].named_parameters():
            arrays["B/" + n] = p.detach().numpy().copy()
        os.chdir(ROOT)
    out = os.path.join(ROOT, "tests", "golden", "trainer.npz")
    np.savez_compressed(out, meta=np.array(json.dumps(meta)), **arrays)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
