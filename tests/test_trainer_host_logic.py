"""CPU: the product `Trainer` on its eager path, `FusedAdamW`'s checkpoint format and device-resident schedule, the schedulers of
`optim.build_lr_scheduler` and `criterion.LossLog`, against what the unmodified reference did (tests/golden/trainer.npz) -- over
tests/fake_device_lib.py, extended here by the two entry points this loop adds."""
import contextlib
import ctypes
import io
import json
import math
import os

import numpy as np
import pytest
import torch

import fake_device_lib
import trainer_stubs as S
from fake_device_lib import f32


class FakeLib(fake_device_lib.FakeLib):
    def mdb_adamw_advance(self, hyper, stream):
        """include/monodetr_b200.h MdbAdamwHyper: doubles t, lr, beta1, beta2, then the float step_size."""
        h = fake_device_lib.f64(hyper, 5)
        t, lr, b1, b2 = float(h[0]) + 1.0, float(h[1]), float(h[2]), float(h[3])
        h[0] = t
        f32(hyper, 10)[8] = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        return 0

    def mdb_trainlog_push_f32(self, values, weights, n, ring, slots, counter, stream):
        c = fake_device_lib.i64(counter, 1)
        rec = f32(ring, slots, n + 1)[int(c[0]) % slots]
        rec[:n] = f32(values, n) * f32(weights, n)
        s = torch.zeros((), dtype=torch.float32)
        for j in range(n):
            s = s + rec[j]
        rec[n] = s
        c[0] += 1
        return 0


@pytest.fixture
def fake(monkeypatch):
    from monodetr_b200 import _lib
    fake_device_lib.install(monkeypatch)
    lib = FakeLib()
    monkeypatch.setattr(_lib, "_lib", lib)
    return lib


@pytest.fixture(scope="module")
def golden(golden_dir):
    z = np.load(os.path.join(golden_dir, "trainer.npz"))
    return json.loads(str(z["meta"])), z


def _train(cfg, tester=None, device_step=False, loader=None):
    from monodetr_b200.optim import build_lr_scheduler, FusedAdamW
    from monodetr_b200.trainer import Trainer
    model = S.StubModel()
    opt = FusedAdamW(model, lr=S.OPT_CFG["lr"], weight_decay=S.OPT_CFG["weight_decay"], device_step=device_step)
    sched, warm = build_lr_scheduler(S.SCHED_CFG, opt, last_epoch=-1)
    logger = S.ListLogger()
    tr = Trainer(cfg, model, opt, loader or S.make_loader(), None, sched, warm, logger, S.StubCriterion(), "stub")
    tr.tester = tester
    lrs, step = [], opt.step

    def counting_step(*a, **k):
        lrs.append([g["lr"] for g in opt.param_groups])
        return step(*a, **k)
    opt.step = counting_step
    np.random.seed(7)
    out = io.StringIO()
    with contextlib.redirect_stdout(out), contextlib.redirect_stderr(io.StringIO()):
        tr.train()
    files = {}
    for f in sorted(os.listdir(tr.output_dir)):
        c = torch.load(os.path.join(tr.output_dir, f), weights_only=False)
        files[f] = [c["epoch"], c["best_result"], c["best_epoch"]]
    return {"lrs": lrs, "stdout": out.getvalue(), "logger": logger.lines, "files": files, "opt": opt, "model": model, "trainer": tr,
            "numpy_seed": int(np.random.get_state()[1][0])}


def _structure(sd):
    return {"state": {str(i): {"step": int(s["step"]), "shapes": {k: list(v.shape) for k, v in s.items() if torch.is_tensor(v)}}
                      for i, s in sd["state"].items()},
            "param_groups": [{k: (list(v) if isinstance(v, (tuple, list)) else v) for k, v in g.items()} for g in sd["param_groups"]]}


@pytest.mark.parametrize("device_step", [False, True])
def test_eager_path_reproduces_the_reference_run(fake, golden, tmp_path, monkeypatch, device_step):
    meta, arrays = golden
    monkeypatch.chdir(tmp_path)
    r = _train(dict(S.CFG), tester=S.StubTester(), device_step=device_step)
    a = meta["A"]
    assert not r["trainer"].graph_path                      # a criterion that is not the device one: the reference's loop
    assert r["lrs"] == a["lrs"]
    assert r["stdout"] == a["stdout"]
    assert r["logger"] == a["logger"]
    assert r["files"] == a["files"]
    assert r["numpy_seed"] == a["numpy_seed"]
    for n, p in r["model"].named_parameters():
        np.testing.assert_allclose(p.detach().numpy(), arrays["A/" + n], rtol=2e-5, atol=1e-6, err_msg=n)
    sd = r["opt"].state_dict()
    assert _structure(sd) == a["state_dict"]
    assert [list(g) for g in sd["param_groups"]] == [list(g) for g in a["state_dict"]["param_groups"]]      # key order too
    for i, s in sd["state"].items():
        np.testing.assert_allclose(s["exp_avg"].numpy(), arrays[f"A/exp_avg/{i}"], rtol=1e-4, atol=1e-7)
        np.testing.assert_allclose(s["exp_avg_sq"].numpy(), arrays[f"A/exp_avg_sq/{i}"], rtol=1e-4, atol=1e-9)
    assert fake.calls["mdb_adamw_step_f32"] == len(a["lrs"])
    assert fake.calls.get("mdb_adamw_advance", 0) == (len(a["lrs"]) if device_step else 0)


def test_resume_continues_the_sequence(fake, golden, tmp_path, monkeypatch):
    meta, arrays = golden
    monkeypatch.chdir(tmp_path)
    cfg = dict(S.CFG, save_all=False, max_epoch=3)
    first = _train(cfg)
    assert first["lrs"] == meta["B"]["first"]["lrs"] and first["files"] == meta["B"]["first"]["files"]
    r = _train(dict(cfg, max_epoch=7, resume_model=True))
    b = meta["B"]["resumed"]
    assert r["lrs"] == b["lrs"] and r["logger"] == b["logger"] and r["files"] == b["files"]
    assert r["opt"].step_count == 7 * S.N_BATCHES
    for n, p in r["model"].named_parameters():
        np.testing.assert_allclose(p.detach().numpy(), arrays["B/" + n], rtol=2e-5, atol=1e-6, err_msg=n)


def _stepped(device_step=False, steps=3):
    from monodetr_b200.optim import FusedAdamW
    model = S.StubModel()
    opt = FusedAdamW(model, lr=1e-2, weight_decay=1e-2, device_step=device_step)
    for _ in range(steps):
        opt.zero_grad()
        model(torch.ones(2, 4), None, None, None)["x"].sum().backward()
        opt.step()
    return model, opt


def test_state_dict_round_trip_and_what_it_refuses(fake):
    from monodetr_b200.optim import FusedAdamW
    model, opt = _stepped()
    sd = opt.state_dict()
    assert sorted(sd["state"]) == [0, 2, 3, 5] and all(s["step"] == 3 for s in sd["state"].values())        # sa_v_proj: no entry
    assert sd["state"][3]["exp_avg"].shape == model.a.weight.shape
    assert sd["state"][3]["exp_avg"].data_ptr() != opt.exp_avg.data_ptr()                                    # copies, not views
    for device_step in (False, True):
        other = FusedAdamW(S.StubModel(), lr=0.5, device_step=device_step)
        assert other.state_dict()["state"] == {}                                                             # nothing before the first step
        loaded = {"state": sd["state"], "param_groups": [dict(g, foreach=None, capturable=False) for g in sd["param_groups"]]}
        other.load_state_dict(loaded)                                                                        # keys of a newer torch: ignored
        assert other.step_count == 3 and torch.equal(other.exp_avg, opt.exp_avg) and torch.equal(other.exp_avg_sq, opt.exp_avg_sq)
        assert [g["lr"] for g in other.param_groups] == [1e-2, 1e-2]
        assert [g["weight_decay"] for g in other.param_groups] == [0, 1e-2]
        if device_step:
            assert float(other._hyper[0]) == 3.0 and float(other._hyper[1]) == 1e-2
    mixed = {"state": {i: dict(s) for i, s in sd["state"].items()}, "param_groups": sd["param_groups"]}
    mixed["state"][2]["step"] = 2
    with pytest.raises(ValueError, match="one step count"):
        opt.load_state_dict(mixed)
    missing = {"state": {i: s for i, s in sd["state"].items() if i != 5}, "param_groups": sd["param_groups"]}
    with pytest.raises(ValueError, match="missing"):
        opt.load_state_dict(missing)
    with pytest.raises(ValueError, match="no gradient"):
        opt.load_state_dict({"state": {**sd["state"], 1: sd["state"][0]}, "param_groups": sd["param_groups"]})
    with pytest.raises(ValueError, match="two groups"):
        opt.load_state_dict({"state": {}, "param_groups": sd["param_groups"][:1]})


def test_reference_adamw_state_loads(fake, golden):
    """The packed dict torch builds for an optimizer over `[biases, weights]` of all named parameters -- the reference's."""
    from monodetr_b200.optim import FusedAdamW
    ref_model = S.StubModel()
    named = list(ref_model.named_parameters())
    ref = torch.optim.Adam([{"params": [p for n, p in named if "bias" in n], "weight_decay": 0},
                            {"params": [p for n, p in named if "bias" not in n], "weight_decay": 0.01}], lr=3e-3)
    for _ in range(2):
        ref.zero_grad()
        ref_model(torch.ones(2, 4), None, None, None)["x"].sum().backward()
        ref.step()
    sd = ref.state_dict()
    assert sorted(sd["state"]) == [0, 2, 3, 5]
    opt = FusedAdamW(S.StubModel(), lr=1.0, weight_decay=0.01)
    opt.load_state_dict(sd)                                                   # step is a tensor here, extra group keys are present
    assert opt.step_count == 2 and opt.param_groups[0]["lr"] == 3e-3
    for off, p, name in zip(opt.bucket.offsets, opt.bucket.params, opt.bucket.names):
        i = [n for n, _ in named if "bias" in n].index(name) if "bias" in name else 3 + [n for n, _ in named if "bias" not in n].index(name)
        assert torch.equal(opt.exp_avg[off:off + p.numel()].view_as(p), sd["state"][i]["exp_avg"])


def test_schedule_reaches_the_device_block(fake):
    """lr written to `param_groups` by a scheduler is what the next device-side step uses; differing group lrs are refused."""
    model, opt = _stepped(device_step=True, steps=1)
    host = lambda lr, t: np.float32(lr * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t))       # noqa: E731
    assert np.float32(opt._step_size.item()) == host(1e-2, 1)
    for g in opt.param_groups:
        g["lr"] = 5e-4
    opt.step()
    assert np.float32(opt._step_size.item()) == host(5e-4, 2) and opt.step_count == 2
    opt.param_groups[0]["lr"] = 1e-3
    with pytest.raises(ValueError, match="one learning rate"):
        opt.step()


def test_loss_log_matches_item(fake):
    from monodetr_b200.criterion import LossLog, NUM_LOSSES, SetCriterion, HungarianMatcher, build_weight_dict
    w = build_weight_dict({"cls_loss_coef": 2, "bbox_loss_coef": 5, "giou_loss_coef": 2, "dim_loss_coef": 1, "angle_loss_coef": 1,
                           "depth_loss_coef": 1, "3dcenter_loss_coef": 10, "depth_map_loss_coef": 1})
    crit = SetCriterion(3, HungarianMatcher(), w, 0.25, ["labels", "boxes", "cardinality", "depths", "dims", "angles", "center", "depth_map"])
    log = LossLog(crit, 3, torch.device("cpu"), slots=4)
    assert len(log.terms) == 8 + 7 + 7 and log.terms[0][0] == "loss_ce" and "class_error" not in dict(log.terms)
    tables = []
    for step in range(6):                                   # wraps around the 4-slot ring
        crit._last_losses = torch.rand(3, NUM_LOSSES) * 3
        tables.append(crit._last_losses.clone())
        log.push()
        got = log.fetch(step).read()
        want, total = {}, 0
        for name, i in log.terms:
            want[name] = (tables[step].reshape(-1)[i] * w[name]).item()
            total += want[name]
        want["loss_detr"] = total
        assert got == want and list(got) == list(want)
    assert log.fetch(3).read()["loss_ce"] == (tables[3][0, 0] * w["loss_ce"]).item()
    with pytest.raises(ValueError, match="no longer in the ring"):
        log.fetch(1)
