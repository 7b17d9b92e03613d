"""CPU: oracle/trainer.py (the reference training loop's control flow in plain Python) reproduces what the unmodified reference
`Trainer` did when tools/gen_golden_trainer.py ran it: tests/golden/trainer.npz."""
import json
import os

import numpy as np
import pytest

import trainer_stubs as S
from oracle import trainer as ot


@pytest.fixture(scope="module")
def golden(golden_dir):
    return json.loads(str(np.load(os.path.join(golden_dir, "trainer.npz"))["meta"]))


def _per_epoch(lrs):
    assert len(lrs) % S.N_BATCHES == 0 and all(len(set(l)) == 1 for l in lrs)              # both groups share the lr
    per = [lrs[i:i + S.N_BATCHES] for i in range(0, len(lrs), S.N_BATCHES)]
    assert all(len({l[0] for l in ep}) == 1 for ep in per)                                # constant within an epoch
    return [ep[0][0] for ep in per]


def test_straight_run_with_tester(golden):
    a = golden["A"]
    sim = ot.simulate(S.CFG, S.SCHED_CFG, S.OPT_CFG["lr"], ap_script=S.AP_SCRIPT)
    assert sim["lrs"] == _per_epoch(a["lrs"])
    assert sim["logger"] == a["logger"]
    assert sim["files"] == a["files"]


def test_resumed_run(golden):
    b = golden["B"]
    cfg = dict(S.CFG, save_all=False, max_epoch=3)
    first = ot.simulate(cfg, S.SCHED_CFG, S.OPT_CFG["lr"])
    assert first["lrs"] == _per_epoch(b["first"]["lrs"]) and first["files"] == b["first"]["files"]
    assert first["logger"] == b["first"]["logger"]
    saved_lr = ot.warmup_lr(S.OPT_CFG["lr"], 3)                                            # the lr the checkpoint of epoch 3 holds
    sim = ot.simulate(dict(cfg, max_epoch=7), S.SCHED_CFG, S.OPT_CFG["lr"], resume=(3, 0, 0, saved_lr))
    assert sim["lrs"] == _per_epoch(b["resumed"]["lrs"])
    assert sim["files"] == b["resumed"]["files"]
    assert sim["logger"] == [l for l in b["resumed"]["logger"] if not l.startswith("==>")]
