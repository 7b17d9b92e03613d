"""CPU: Tester.test() (tester_helper.py:26-63) -- which checkpoint files it picks in 'single' and 'all' mode, their order, and
its errors -- with a stub model and a Tester whose inference() / evaluate() only record which weights they saw."""
import os

import pytest
import torch

from monodetr_b200 import tester, trainer
from trainer_stubs import StubModel


class Log:
    def __init__(self):
        self.lines = []

    def info(self, s):
        self.lines.append(s)


class RecordingTester(tester.Tester):
    """Tester.test() as written, around a model on the CPU; inference() / evaluate() log the epoch stored in the weights."""

    def __init__(self, cfg, output_dir, save_all):
        self.cfg, self.train_cfg = cfg, {"save_all": save_all, "save_path": "unused"}
        self.model, self.logger, self.output_dir = StubModel(), Log(), str(output_dir)
        self.device = torch.device("cpu")
        self.seen = []

    def inference(self):
        self.logger.info("inference")

    def evaluate(self):
        self.seen.append(int(round(float(self.model.a.bias.detach()[0]))))
        self.logger.info("evaluate")
        return 0.0


def write(out, name, epoch, mtime=None):
    """A checkpoint in the Trainer's format whose weights record `epoch`."""
    model = StubModel()
    with torch.no_grad():
        model.a.bias[0] = epoch
    os.makedirs(out, exist_ok=True)
    trainer.save_checkpoint(trainer.get_checkpoint_state(model, None, epoch, 0.0, 0), os.path.join(out, name))
    if mtime is not None:
        os.utime(os.path.join(out, name + ".pth"), (mtime, mtime))


@pytest.fixture
def out(tmp_path):
    d = tmp_path / "monodetr"
    t0 = 1_700_000_000
    for e in range(1, 6):
        write(d, f"checkpoint_epoch_{e}", e, t0 + 10 * e)
    write(d, "checkpoint_best", 100, t0 + 100)
    write(d, "checkpoint", 200, t0 + 200)
    return d


@pytest.mark.parametrize("mode", ["single", "all"])
def test_single_checkpoint_without_save_all_is_the_best(out, mode):
    t = RecordingTester({"mode": mode, "checkpoint": 3}, out, save_all=False)
    assert t.test() is None
    assert t.seen == [100]
    path = os.path.join(str(out), "checkpoint_best.pth")
    assert t.logger.lines == ["==> Loading from checkpoint '{}'".format(path), "==> Done", "inference", "evaluate"]


def test_single_checkpoint_with_save_all_is_the_named_epoch(out):
    t = RecordingTester({"mode": "single", "checkpoint": 3}, out, save_all=True)
    t.test()
    assert t.seen == [3]
    assert t.logger.lines[0] == "==> Loading from checkpoint '{}'".format(os.path.join(str(out), "checkpoint_epoch_3.pth"))


def test_all_checkpoints_from_the_start_epoch_in_mtime_order(out):
    t0 = 1_700_000_000
    os.utime(out / "checkpoint_epoch_4.pth", (t0, t0))                      # oldest file first, whatever its epoch
    write(out, "checkpoint_epoch_12", 12, t0 + 55)
    (out / "sub").mkdir()
    write(out / "sub", "checkpoint_epoch_9", 9, t0 + 1)                     # not directly in output_dir
    (out / "checkpoint_epoch_x.pth").write_bytes(b"")                       # not an epoch checkpoint's name
    (out / "notes.txt").write_text("x")
    t = RecordingTester({"mode": "all", "checkpoint": "3"}, out, save_all=True)
    t.test()
    assert t.seen == [4, 3, 5, 12]                                          # best / last / epochs < 3 skipped
    assert sum(s.startswith("==> Loading from checkpoint") for s in t.logger.lines) == 4


def test_all_checkpoints_equal_mtimes_follow_the_epoch(out):
    for e in range(1, 6):
        os.utime(out / f"checkpoint_epoch_{e}.pth", (1_700_000_000, 1_700_000_000))
    t = RecordingTester({"mode": "all", "checkpoint": 0}, out, save_all=True)
    t.test()
    assert t.seen == [1, 2, 3, 4, 5]


def test_all_checkpoints_of_a_missing_directory_is_nothing(tmp_path):
    t = RecordingTester({"mode": "all", "checkpoint": 0}, tmp_path / "none", save_all=True)
    assert t.test() is None and t.seen == [] and t.logger.lines == []


@pytest.mark.parametrize("cfg", [{"mode": "best", "checkpoint": 1}, {"checkpoint": 1}, {"mode": None}])
def test_bad_mode_raises(out, cfg):
    t = RecordingTester(cfg, out, save_all=True)
    with pytest.raises(ValueError, match="'single' or 'all'"):
        t.test()
    assert t.seen == []


def test_missing_checkpoint_names_the_path(out, tmp_path):
    t = RecordingTester({"mode": "single", "checkpoint": 7}, out, save_all=True)
    with pytest.raises(FileNotFoundError, match="checkpoint_epoch_7.pth"):
        t.test()
    os.remove(out / "checkpoint_best.pth")
    t = RecordingTester({"mode": "single", "checkpoint": 7}, out, save_all=False)
    with pytest.raises(FileNotFoundError, match="checkpoint_best.pth"):
        t.test()
    assert t.seen == []


def test_reference_layout_checkpoint_loads(out):
    """A checkpoint as the reference's save_helper writes it (plain model_state, no 'module.' prefix, optimizer_state None)."""
    model = StubModel()
    with torch.no_grad():
        model.a.bias[0] = 42
    torch.save({"epoch": 42, "model_state": model.state_dict(), "optimizer_state": None, "best_result": 0.5, "best_epoch": 42},
               out / "checkpoint_epoch_42.pth")
    t = RecordingTester({"mode": "single", "checkpoint": 42}, out, save_all=True)
    t.test()
    assert t.seen == [42]
