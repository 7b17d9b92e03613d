"""GPU: Tester.test() with the small golden model -- each mode writes the result files and logs the AP that load_state_dict +
inference() + evaluate() give on a freshly built model, and a checkpoint evaluated after another one gives, byte for byte, what
it gives on its own (no weight-derived cache outlives load_state_dict), in both error-compensated precision modes."""
import os
import types

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib, tc, tester, trainer
from monodetr_b200 import kitti_eval as ke
from oracle import monodetr_torch as om
from test_validation_gpu import NAMES, Log, _Loader, labels_near, write_file_path

pytestmark = pytest.mark.gpu
IDS = [3, 8, 15, 16, 42, 77]
MEAN = np.zeros((3, 3), np.float32)


def state_a():
    return om.with_aliases(om.deterministic_state_dict())


def state_b():
    """A seeded perturbation of every floating tensor (frozen BatchNorm statistics included), signs kept."""
    base = om.deterministic_state_dict()
    g = torch.Generator().manual_seed(1234)
    out = {k: (v * torch.exp(0.05 * torch.randn(v.shape, generator=g)) if v.is_floating_point() else v.clone())
           for k, v in base.items()}
    return om.with_aliases(out)


def build(state):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG))
    model.load_state_dict(state)
    return model.cuda().eval()


@pytest.fixture(scope="module")
def setup(tmp_path_factory):
    """Batches of the small golden model's inputs and labels near checkpoint A's detections."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "model_eval_small.npz"))
    images, calibs, sizes = om.synthetic_inputs(len(IDS), int(g["seed"]), H=int(g["H"]), W=int(g["W"]))
    B = 2
    batches = [(images[b:b + B], calibs[b:b + B], {}, {"img_id": torch.tensor(IDS[b:b + B]), "img_size": sizes[b:b + B]})
               for b in range(0, len(IDS), B)]
    root = tmp_path_factory.mktemp("tester_ckpt")
    model = build(state_a())
    with torch.no_grad():
        outs = [model(x.cuda(), c.cuda(), None, s["img_size"].cuda()) for x, c, _, s in batches]
    write_file_path(str(root / "ref"), [(o, s["img_size"].cuda(), c.cuda()) for o, (_, c, _, s) in zip(outs, batches)],
                    [IDS[b:b + B] for b in range(0, len(IDS), B)], MEAN, thr=0.0)
    os.makedirs(root / "label_2")
    for i, text in zip(IDS, labels_near(ke.get_label_annos(str(root / "ref")), np.random.default_rng(2))):
        (root / "label_2" / ("%06d.txt" % i)).write_text(text)
    ds = types.SimpleNamespace(idx_list=["%06d" % i for i in IDS], label_dir=str(root / "label_2"), writelist=["Car"],
                               class_name=NAMES, cls_mean_size=MEAN, split="val", max_objs=50)
    return types.SimpleNamespace(batches=batches, ds=ds)


def make_tester(setup, model, save_path, cfg=None):
    cfg = dict({"topk": 50, "threshold": 0.0}, **(cfg or {}))
    return tester.Tester(cfg, model, _Loader(setup.ds, setup.batches), Log(), {"save_path": save_path, "save_all": True})


def result_files(t):
    d = os.path.join(t.output_dir, "outputs", "data")
    return {i: open(os.path.join(d, "%06d.txt" % i), "rb").read() for i in IDS}


def fresh(setup, state, tmp_path, tag):
    """load_state_dict + inference() + evaluate() on a freshly built model: (AP, log lines, result files)."""
    t = make_tester(setup, build(state), f"fresh_{tag}/")
    was = torch.is_grad_enabled()
    try:
        t.inference()
        ap = t.evaluate()
    finally:
        torch.set_grad_enabled(was)
    return ap, t.logger.lines, result_files(t)


def write_checkpoints(out, model_for_states):
    """checkpoint_epoch_1 = A, checkpoint_epoch_2 = B (newer), checkpoint_best = B, written by the Trainer's save path."""
    os.makedirs(out, exist_ok=True)
    for epoch, name, state in ((1, "checkpoint_epoch_1", state_a()), (2, "checkpoint_epoch_2", state_b()),
                               (2, "checkpoint_best", state_b())):
        model_for_states.load_state_dict(state)
        trainer.save_checkpoint(trainer.get_checkpoint_state(model_for_states, None, epoch, 0.5, 2), os.path.join(out, name))
    t0 = 1_700_000_000
    for k, name in enumerate(("checkpoint_epoch_1", "checkpoint_epoch_2", "checkpoint_best")):
        os.utime(os.path.join(out, name + ".pth"), (t0 + k, t0 + k))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
def test_checkpoints_evaluate_as_a_fresh_model(setup, tmp_path, monkeypatch, precision):
    monkeypatch.chdir(tmp_path)
    was_prec, was_det = tc.get_precision(), _lib.deterministic()
    tc.set_precision(precision)
    _lib.lib().mdb_set_deterministic(1)            # byte-for-byte comparisons of whole evaluation passes
    was_grad = torch.is_grad_enabled()
    try:
        ref_a = fresh(setup, state_a(), tmp_path, "a")
        ref_b = fresh(setup, state_b(), tmp_path, "b")
        assert ref_a[2] != ref_b[2]                                            # the two checkpoints detect differently
        model = build(state_a())
        out = os.path.join("out", "monodetr")
        write_checkpoints(out, model)

        def load_lines(name):
            path = os.path.join("./out/", "monodetr", name)
            return ["==> Loading from checkpoint '{}'".format(path), "==> Done"]

        # 'all': A then B with the same model object; B's pass is what a fresh model gives for B
        model.load_state_dict(state_a())
        t = make_tester(setup, model, "out/", {"mode": "all", "checkpoint": 0})
        assert t.test() is None
        assert t.logger.lines == load_lines("checkpoint_epoch_1.pth") + ref_a[1] + load_lines("checkpoint_epoch_2.pth") + ref_b[1]
        assert result_files(t) == ref_b[2]
        # 'single' with save_all: the named epoch (A after B, on the same model)
        t = make_tester(setup, model, "out/", {"mode": "single", "checkpoint": 1})
        t.test()
        assert t.logger.lines == load_lines("checkpoint_epoch_1.pth") + ref_a[1]
        assert result_files(t) == ref_a[2]
        # 'single' without save_all: checkpoint_best (B)
        t = make_tester(setup, model, "out/", {"mode": "single", "checkpoint": 1})
        t.train_cfg["save_all"] = False
        t.test()
        assert t.logger.lines == load_lines("checkpoint_best.pth") + ref_b[1]
        assert result_files(t) == ref_b[2]
        # the AP each pass logs is the one evaluate() returns on the fresh model
        assert ref_b[0] == t.evaluate()
    finally:
        torch.set_grad_enabled(was_grad)
        tc.set_precision(was_prec)
        _lib.lib().mdb_set_deterministic(int(was_det))


def test_reference_layout_checkpoint_loads(setup, tmp_path, monkeypatch):
    """A checkpoint as the reference's save_helper writes it for a model that is not wrapped: model_state without a 'module.'
    prefix, the reference's own key names (aliases included), optimizer_state None."""
    monkeypatch.chdir(tmp_path)
    was_det, was_grad = _lib.deterministic(), torch.is_grad_enabled()
    _lib.lib().mdb_set_deterministic(1)
    try:
        ref_b = fresh(setup, state_b(), tmp_path, "b")
        os.makedirs(os.path.join("out", "monodetr"))
        sd = state_b()
        assert not any(k.startswith("module.") for k in sd)
        torch.save({"epoch": 7, "model_state": sd, "optimizer_state": None, "best_result": 0.1, "best_epoch": 7},
                   os.path.join("out", "monodetr", "checkpoint_epoch_7.pth"))
        t = make_tester(setup, build(state_a()), "out/", {"mode": "single", "checkpoint": 7})
        t.test()
        assert t.logger.lines[2:] == ref_b[1]
        assert result_files(t) == ref_b[2]
    finally:
        torch.set_grad_enabled(was_grad)
        _lib.lib().mdb_set_deterministic(int(was_det))
