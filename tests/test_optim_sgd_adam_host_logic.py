"""CPU: `FusedSGD` / `FusedAdam` (monodetr_b200/optim.py) -- the reference's `sgd` and `adam` optimizer types -- against
torch.optim.SGD / torch.optim.Adam over `trainer_stubs.StubModel`: `build_optimizer`'s routing, the update, the checkpoint
format in both directions, what `load_state_dict` refuses, the `Trainer` path each one takes, and the new C-ABI symbols.  The
four entry points are restated below in torch CPU operations, in the kernels' order."""
import contextlib
import ctypes
import io
import os

import numpy as np
import pytest
import torch

import fake_device_lib
import trainer_stubs as S
from fake_device_lib import f32, f64

KINDS = ("sgd", "adam")


class FakeLib(fake_device_lib.FakeLib):
    def mdb_sgd_advance(self, hyper, stream):
        """include/monodetr_b200.h MdbSgdHyper: doubles t, lr."""
        f64(hyper, 2)[0] += 1.0
        return 0

    def mdb_sgd_step_f32(self, p, g, buf, n, n_decay, momentum, wd, lr, first, hyper, stream):
        P, G, B = f32(p, n), f32(g, n), f32(buf, n)
        if hyper:
            h = f64(hyper, 2)
            lr, first = float(h[1]), float(h[0]) == 1.0
        decay = torch.zeros(n)
        decay[:n_decay] = wd
        d = G + decay * P
        if first:
            B.copy_(d)
        else:
            B.mul_(momentum).add_(d)
        P.add_(B, alpha=-lr)
        return 0

    def mdb_adam_advance(self, hyper, stream):
        """MdbAdamHyper: doubles t, lr, beta1, beta2, then the floats neg_step, bc2_sqrt."""
        h = f64(hyper, 5)
        t, lr, b1, b2 = float(h[0]) + 1.0, float(h[1]), float(h[2]), float(h[3])
        h[0] = t
        f32(hyper, 10)[8] = (lr / (1 - b1 ** t)) * -1
        f32(hyper, 10)[9] = (1 - b2 ** t) ** 0.5
        return 0

    def mdb_adam_step_f32(self, p, g, m, v, n, n_decay, omb1, beta2, omb2, eps, wd, neg_step, bc2_sqrt, hyper, stream):
        P, G, M, V = f32(p, n), f32(g, n), f32(m, n), f32(v, n)
        if hyper:
            neg_step, bc2_sqrt = (float(x) for x in f32(hyper, 10)[8:10])
        decay = torch.zeros(n)
        decay[:n_decay] = wd
        gd = G + decay * P
        M.lerp_(gd, omb1)
        V.mul_(beta2).addcmul_(gd, gd, value=omb2)
        P.addcdiv_(M, (V.sqrt() / bc2_sqrt).add_(eps), value=neg_step)
        return 0


@pytest.fixture
def fake(monkeypatch):
    from monodetr_b200 import _lib
    fake_device_lib.install(monkeypatch)
    lib = FakeLib()
    monkeypatch.setattr(_lib, "_lib", lib)
    return lib


def _reference(kind, model, lr=1e-2, wd=1e-2):
    """lib/helpers/optimizer_helper.py:7-27 over the model's named parameters: biases (no decay), then weights."""
    named = list(model.named_parameters())
    groups = [{"params": [p for n, p in named if "bias" in n], "weight_decay": 0},
              {"params": [p for n, p in named if "bias" not in n], "weight_decay": wd}]
    return torch.optim.SGD(groups, lr=lr, momentum=0.9) if kind == "sgd" else torch.optim.Adam(groups, lr=lr)


def _fused(kind, model, lr=1e-2, wd=1e-2, device_step=False):
    from monodetr_b200.optim import FusedAdam, FusedSGD
    if kind == "sgd":
        return FusedSGD(model, lr=lr, momentum=0.9, weight_decay=wd, device_step=device_step)
    return FusedAdam(model, lr=lr, weight_decay=wd, device_step=device_step)


def _step(model, opt, i):
    opt.zero_grad()
    model(torch.ones(2, 4) * (1 + 0.3 * i), None, None, None)["x"].pow(2).sum().backward()
    opt.step()


def _assert_same_state(sd, ref_sd, rtol=1e-5):
    assert sd["param_groups"] == ref_sd["param_groups"]
    assert [list(g) for g in sd["param_groups"]] == [list(g) for g in ref_sd["param_groups"]]          # key order too
    assert list(sd["state"]) == list(ref_sd["state"])
    for i, s in ref_sd["state"].items():
        assert list(sd["state"][i]) == list(s), i
        for k, v in s.items():
            got = sd["state"][i][k]
            assert torch.is_tensor(got) and got.dtype == v.dtype and got.shape == v.shape, (i, k)
            if k == "step":
                assert torch.equal(got, v)
            else:
                torch.testing.assert_close(got, v, rtol=rtol, atol=1e-7)


def test_build_optimizer_routes_every_reference_type(fake):
    from monodetr_b200.optim import FusedAdam, FusedAdamW, FusedSGD, build_optimizer
    for kind, cls in (("adamw", FusedAdamW), ("sgd", FusedSGD), ("adam", FusedAdam)):
        opt = build_optimizer({"type": kind, "lr": 3e-3, "weight_decay": 0.05}, S.StubModel())
        assert type(opt) is cls and not opt.device_step
        assert [g["weight_decay"] for g in opt.param_groups] == [0, 0.05] and [g["lr"] for g in opt.param_groups] == [3e-3] * 2
        nd = len(opt.param_groups[1]["params"])
        assert all("bias" in n for n in opt.bucket.names[nd:]) and not any("bias" in n for n in opt.bucket.names[:nd])
    assert build_optimizer({"type": "sgd", "lr": 1.0, "weight_decay": 0}, S.StubModel()).param_groups[1]["momentum"] == 0.9
    with pytest.raises(NotImplementedError, match="rmsprop optimizer is not supported"):
        build_optimizer({"type": "rmsprop", "lr": 1.0, "weight_decay": 0}, S.StubModel())


@pytest.mark.parametrize("device_step", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_update_and_state_dict_equal_torch(fake, kind, device_step):
    ref_model, model = S.StubModel(), S.StubModel()
    ref, opt = _reference(kind, ref_model), _fused(kind, model, device_step=device_step)
    assert opt.state_dict() == {"state": {}, "param_groups": ref.state_dict()["param_groups"]}          # nothing before a step
    for i in range(4):
        _step(ref_model, ref, i)
        _step(model, opt, i)
    assert opt.step_count == 4
    for (n, p), (_, q) in zip(model.named_parameters(), ref_model.named_parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-5, atol=1e-7, msg=n)
    assert torch.equal(model.sa_v_proj.weight, S.StubModel().sa_v_proj.weight)                         # no gradient: untouched
    sd = opt.state_dict()
    _assert_same_state(sd, ref.state_dict())
    assert sorted(sd["state"]) == [0, 2, 3, 5]
    key = "momentum_buffer" if kind == "sgd" else "exp_avg"
    assert sd["state"][3][key].data_ptr() != getattr(opt, key).data_ptr()                              # copies, not views
    assert fake.calls.get("mdb_%s_advance" % kind, 0) == (4 if device_step else 0)
    assert fake.calls["mdb_%s_step_f32" % kind] == 4


@pytest.mark.parametrize("device_step", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_torch_state_loads_and_continues(fake, kind, device_step):
    """A state torch saved -- after two steps, and before any (no momentum buffers / moments yet) -- continues on torch's path."""
    for taken in (2, 0):
        ref_model = S.StubModel()
        ref = _reference(kind, ref_model, lr=3e-3)
        for i in range(taken):
            _step(ref_model, ref, i)
        model = S.StubModel()
        model.load_state_dict(ref_model.state_dict())
        opt = _fused(kind, model, lr=0.5, device_step=device_step)
        opt.load_state_dict(ref.state_dict())
        assert [g["lr"] for g in opt.param_groups] == [3e-3, 3e-3]
        assert opt.step_count == (0 if taken == 0 else (1 if kind == "sgd" else taken))
        for i in range(taken, taken + 2):
            _step(ref_model, ref, i)
            _step(model, opt, i)
        for (n, p), (_, q) in zip(model.named_parameters(), ref_model.named_parameters()):
            torch.testing.assert_close(p.detach(), q.detach(), rtol=1e-5, atol=1e-7, msg=(taken, n))
        if kind == "adam":
            _assert_same_state(opt.state_dict(), ref.state_dict())
        else:
            torch.testing.assert_close(opt.state_dict()["state"][3]["momentum_buffer"], ref.state_dict()["state"][3]["momentum_buffer"])
        # and the other way: the fused state loads into torch's optimizer
        back = _reference(kind, S.StubModel())
        back.load_state_dict(opt.state_dict())
        _assert_same_state(back.state_dict(), opt.state_dict())


@pytest.mark.parametrize("kind", KINDS)
def test_what_load_state_dict_and_step_refuse(fake, kind):
    model = S.StubModel()
    opt = _fused(kind, model)
    for i in range(2):
        _step(model, opt, i)
    sd = opt.state_dict()
    missing = {"state": {i: s for i, s in sd["state"].items() if i != 5}, "param_groups": sd["param_groups"]}
    with pytest.raises(ValueError, match="missing"):
        opt.load_state_dict(missing)
    with pytest.raises(ValueError, match="no gradient"):
        opt.load_state_dict({"state": {**sd["state"], 1: sd["state"][0]}, "param_groups": sd["param_groups"]})
    with pytest.raises(ValueError, match="two groups"):
        opt.load_state_dict({"state": {}, "param_groups": sd["param_groups"][:1]})
    unsupported = ("nesterov", True) if kind == "sgd" else ("amsgrad", True)
    for key, value in (unsupported, ("maximize", True)) + ((("dampening", 0.1),) if kind == "sgd" else (("decoupled_weight_decay", True),)):
        with pytest.raises(ValueError, match="not supported"):
            opt.load_state_dict({"state": sd["state"], "param_groups": [dict(g, **{key: value}) for g in sd["param_groups"]]})
    if kind == "adam":
        mixed = {"state": {i: dict(s) for i, s in sd["state"].items()}, "param_groups": sd["param_groups"]}
        mixed["state"][2]["step"] = torch.tensor(1.0)
        with pytest.raises(ValueError, match="one step count"):
            opt.load_state_dict(mixed)
    opt.load_state_dict(sd)                                                  # the refusals changed nothing that matters
    opt.param_groups[0]["lr"] = 1e-3
    with pytest.raises(ValueError, match="one learning rate"):
        opt.step()
    with pytest.raises(ValueError):
        _fused(kind, S.StubModel(), lr=-1.0)
    if kind == "sgd":
        from monodetr_b200.optim import FusedSGD
        with pytest.raises(ValueError, match="momentum"):
            FusedSGD(S.StubModel(), lr=1.0, momentum=0.0)


@pytest.mark.parametrize("kind", KINDS)
def test_trainer_paths_and_checkpoints(fake, kind, tmp_path, monkeypatch):
    """The `Trainer`'s eager loop with a fused optimizer follows the same loop with torch's, and writes checkpoints torch loads;
    the graph path is chosen for a fused optimizer with `device_step=True` and the device criterion only."""
    from monodetr_b200.criterion import HungarianMatcher, SetCriterion
    from monodetr_b200.optim import build_lr_scheduler
    from monodetr_b200.trainer import Trainer
    monkeypatch.chdir(tmp_path)
    cfg = dict(S.CFG, max_epoch=3, save_all=False)
    runs = {}
    for name in ("fused", "torch"):
        model = S.StubModel()
        opt = _fused(kind, model) if name == "fused" else _reference(kind, model)
        sched, warm = build_lr_scheduler(S.SCHED_CFG, opt, last_epoch=-1)
        tr = Trainer(cfg, model, opt, S.make_loader(), None, sched, warm, S.ListLogger(), S.StubCriterion(), name)
        assert not tr.graph_path
        np.random.seed(7)
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            tr.train()
        runs[name] = (model, opt, torch.load(os.path.join(tr.output_dir, "checkpoint.pth"), weights_only=False))
    (model, opt, ck), (ref_model, ref, ref_ck) = runs["fused"], runs["torch"]
    for (n, p), (_, q) in zip(model.named_parameters(), ref_model.named_parameters()):
        torch.testing.assert_close(p.detach(), q.detach(), rtol=2e-5, atol=1e-6, msg=n)
    _assert_same_state(ck["optimizer_state"], ref_ck["optimizer_state"], rtol=2e-5)
    crit = SetCriterion(3, HungarianMatcher(), {"loss_ce": 1.0}, 0.25, ["labels"])
    for opt, want in ((_fused(kind, S.StubModel(), device_step=True), True), (_fused(kind, S.StubModel()), False),
                      (_reference(kind, S.StubModel()), False)):
        assert Trainer(cfg, S.StubModel(), opt, [], None, None, None, S.ListLogger(), crit, "m").graph_path == want


def test_new_entry_points_are_exported():
    from monodetr_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "run `python -m monodetr_b200.build` first"
    L = ctypes.CDLL(_lib.LIB_PATH)
    arity = {"mdb_sgd_step_f32": 11, "mdb_sgd_advance": 2, "mdb_adam_step_f32": 15, "mdb_adam_advance": 2}
    for name, n in arity.items():
        assert hasattr(L, name) and len(_lib.SIGNATURES[name]) == n, name
