"""GPU: the training loop on the device -- `FusedAdamW`'s device-resident schedule (`mdb_adamw_advance`), its checkpoint format,
`criterion.LossLog` (`mdb_trainlog_push_f32`) and `trainer.Trainer` replaying the whole iteration as a CUDA graph, held bit for
bit (reproducible mode) to the same `Trainer` running the reference's eager loop.  Small shapes: batch 2 at 320x96.
The synchronisation check covers the trainer's own code; a loader that blocks the host is outside it."""
import copy
import math
import os

import numpy as np
import pytest
import torch

import monodetr_b200
import trainer_stubs as S
from monodetr_b200 import kernels as K
from oracle.optim import adamw_reference_step

pytestmark = pytest.mark.gpu


@pytest.fixture
def repro():
    prev = monodetr_b200.set_deterministic(True)
    try:
        yield
    finally:
        monodetr_b200.set_deterministic(prev)


# ---- the optimizer ------------------------------------------------------------------------------------------------------------
def _toy(seed=0):
    torch.manual_seed(seed)
    return torch.nn.ModuleDict({"a": torch.nn.Linear(37, 19), "norm": torch.nn.LayerNorm(19), "sa_v_proj": torch.nn.Linear(3, 3),
                                "b": torch.nn.Linear(19, 3)}).cuda()


def _fused(device_step, seed=0, lr=2e-4):
    from monodetr_b200.optim import FusedAdamW
    model = _toy(seed)
    opt = FusedAdamW(model, lr=lr, weight_decay=1e-4, device_step=device_step)
    g = torch.Generator(device="cuda").manual_seed(1)
    for p in opt.bucket.params:
        p.grad = torch.randn(p.shape, device="cuda", generator=g)
    return model, opt


def _set_lr(opt, lr):
    for g in opt.param_groups:
        g["lr"] = lr


def test_schedule_reaches_a_replayed_graph():
    lrs = [2e-4, 2e-4, 5e-5, 5e-5]
    _, ref = _fused(False)
    for lr in lrs:
        _set_lr(ref, lr)
        ref.step()
    results = []
    for change in (True, False):
        _, opt = _fused(True)
        opt.step()                                          # warm-up step (lr 2e-4)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            opt.step()
        graph.replay()                                      # step 2, lr 2e-4
        if change:
            _set_lr(opt, 5e-5)
            opt.sync_hyper()
        graph.replay()
        graph.replay()
        torch.cuda.synchronize()
        assert opt.step_count == 4
        results.append(opt)
    changed, unchanged = results
    assert torch.equal(changed.flat_p, ref.flat_p) and torch.equal(changed.exp_avg_sq, ref.exp_avg_sq)
    assert not torch.equal(unchanged.flat_p, ref.flat_p)


def test_device_step_size_equals_the_host_value():
    from monodetr_b200 import _lib
    _, opt = _fused(True, lr=2e-4)
    ts = list(range(1, 2001)) + [4999, 10 ** 4, 123457, 10 ** 6, 5 * 10 ** 6]
    out = torch.zeros(len(ts), device="cuda")
    for i, t in enumerate(ts):
        if t > 2000:
            opt.step_count = t - 1
        _lib.call("mdb_adamw_advance", opt._hyper)
        out[i].copy_(opt._step_size[0])
    assert opt.step_count == ts[-1]
    host = np.array([np.float32(2e-4 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)) for t in ts], np.float32)
    got = out.cpu().numpy()
    bad = [(t, float(h), float(g)) for t, h, g in zip(ts, host, got) if h != g]
    assert not bad, bad


def test_state_dict_against_the_reference_update():
    """FusedAdamW -> state_dict -> a CPU optimizer stepping by oracle.optim.adamw_reference_step, and back."""
    from monodetr_b200.optim import FusedAdamW
    model, opt = _fused(True)
    for _ in range(3):
        opt.step()
    sd = opt.state_dict()
    named = list(model.named_parameters())
    order = [n for n, _ in named if "bias" in n] + [n for n, _ in named if "bias" not in n]
    names = opt.bucket.names
    idx = [order.index(n) for n in names]
    assert sorted(sd["state"]) == sorted(idx) and all(sd["state"][i]["step"] == 3 for i in idx)
    assert not any("sa_v_proj" in order[i] for i in sd["state"])
    ps = [p.detach().cpu().clone() for p in opt.bucket.params]
    gs = [p.grad.cpu() for p in opt.bucket.params]
    ms, vs = [sd["state"][i]["exp_avg"].cpu() for i in idx], [sd["state"][i]["exp_avg_sq"].cpu() for i in idx]
    wds = [0.0 if "bias" in n else 1e-4 for n in names]
    adamw_reference_step(ps, gs, ms, vs, 4, 2e-4, 0.9, 0.999, 1e-8, wds)
    opt.step()
    for p, r, n in zip(opt.bucket.params, ps, names):
        assert torch.allclose(p.detach().cpu(), r, rtol=4e-7, atol=1e-9), n
    # the oracle's state -> load_state_dict -> one more step on both
    model2 = _toy()
    opt2 = FusedAdamW(model2, lr=1.0, weight_decay=1e-4, device_step=True)
    with torch.no_grad():
        for p, r in zip(opt2.bucket.params, ps):
            p.copy_(r)
    loaded = {"state": {i: {"step": 4, "exp_avg": m.clone(), "exp_avg_sq": v.clone()} for i, m, v in zip(idx, ms, vs)},
              "param_groups": sd["param_groups"]}
    opt2.load_state_dict(loaded)
    assert opt2.step_count == 4 and opt2.param_groups[0]["lr"] == 2e-4
    for p, g in zip(opt2.bucket.params, gs):
        p.grad = g.cuda()
    opt2.step()
    adamw_reference_step(ps, gs, ms, vs, 5, 2e-4, 0.9, 0.999, 1e-8, wds)
    for p, r, n in zip(opt2.bucket.params, ps, names):
        assert torch.allclose(p.detach().cpu(), r, rtol=4e-7, atol=1e-9), n


# ---- the loss log -------------------------------------------------------------------------------------------------------------
def test_loss_log_in_a_graph_equals_item():
    from bench_extras import CRIT_CFG
    from monodetr_b200.criterion import LossLog, NUM_LOSSES, build_criterion
    crit = build_criterion(CRIT_CFG)
    table = torch.zeros(3, NUM_LOSSES, device="cuda")
    crit._last_losses = table
    log = LossLog(crit, 3, torch.device("cuda"), slots=4)
    log.push()                                              # eager: record 0 (and the weight table is built outside the capture)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        log.push()
    assert log.pushed == 1
    g = torch.Generator(device="cuda").manual_seed(5)
    for step in range(1, 7):
        table.copy_(torch.rand(3, NUM_LOSSES, device="cuda", generator=g) * 7)
        graph.replay()
        log.replayed()
        rec = log.fetch(step)
        want, total = {}, 0
        for name, i in log.terms:
            want[name] = (table.reshape(-1)[i] * crit.weight_dict[name]).item()
            total += want[name]
        want["loss_detr"] = total
        assert rec.read() == want and rec.ready()
    assert int(log.counter.item()) == 7


# ---- the trainer --------------------------------------------------------------------------------------------------------------
H, W = 96, 320
CFG = {"max_epoch": 3, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": "out"}
SCHED = {"warmup": False, "decay_rate": 0.5, "decay_list": [1, 2]}


def _loader(sizes=(2, 2, 2, 1)):
    from bench_extras import synthetic_targets
    from oracle import monodetr_torch as om
    out = []
    for i, b in enumerate(sizes):
        images, calibs, img_sizes = om.synthetic_inputs(b, 40 + i, H=H, W=W)
        targets = {k: v.cuda() for k, v in synthetic_targets(50 + i, b).items()}
        targets["img_size"] = img_sizes.cuda()
        out.append((images.cuda(), calibs.cuda(), targets, {}))
    return out


def _build(cfg, dropout=0.1, tester=None, env_no_graph=False, max_graphs=None):
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr, tc
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    from monodetr_b200.trainer import Trainer
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, dropout=dropout))
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    crit.depth_map_scale = (W // 16, H // 16)
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler(SCHED, opt, last_epoch=-1)
    if env_no_graph:
        os.environ["MDB_NO_GRAPH"] = "1"
    try:
        tr = Trainer(cfg, model, opt, _loader(), None, sched, warm, S.ListLogger(), crit, "m")
    finally:
        os.environ.pop("MDB_NO_GRAPH", None)
    if max_graphs is not None:
        tr.MAX_GRAPHS = max_graphs
    tr.PRINT_EVERY = 1
    tr.tester = tester
    K.reseed(torch.device("cuda", torch.cuda.current_device()), 4242)      # the key the model's device has
    return tr


def _state(tr):
    opt = tr.optimizer
    return [opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), torch.tensor(float(opt.step_count))] + \
        [p.detach().clone() for p in tr.model.parameters()]


def _epochs(tr, n, logs):
    """`train()`'s body per epoch without the files; returns the state after every epoch."""
    states = []
    for epoch in range(n):
        tr.train_one_epoch(epoch)
        tr.epoch += 1
        tr.lr_scheduler.step()
        tr.optimizer.sync_hyper()
        states.append(_state(tr))
    return states


def test_graph_path_equals_eager_path(repro, monkeypatch, capsys):
    from monodetr_b200 import trainer as T
    runs = {}
    for name, kw in (("graph", {}), ("eager_device_step", {"max_graphs": 0}), ("reference_loop", {"env_no_graph": True})):
        logs = []
        monkeypatch.setattr(T, "print_losses", lambda i, log, logs=logs: logs.append((i, dict(log))))
        tr = _build(CFG, **kw)
        assert tr.graph_path == (name != "reference_loop")
        live = []
        if name == "graph":
            replay = torch.cuda.CUDAGraph.replay
            monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (live.append(tr.live_graphs), replay(g))[1])
        states = _epochs(tr, 3, logs)
        if name == "graph":
            monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", replay)
            # epoch 0: batch 0 eager, 1-2 replayed, the short one eager; afterwards everything replayed
            assert len(live) == 2 + 4 + 4 and max(live) == 2 and tr.live_graphs == 2
        assert tr.optimizer.step_count == 12 and [g["lr"] for g in tr.optimizer.param_groups] == [2e-4 * 0.25] * 2
        runs[name] = (states, logs)
    g_states, g_logs = runs["graph"]
    assert len(g_logs) == 12 and len(g_logs[0][1]) == 8 + 7 + 7 + 1
    for other in ("eager_device_step", "reference_loop"):
        o_states, o_logs = runs[other]
        for e, (a, b) in enumerate(zip(g_states, o_states)):
            bad = [i for i, (x, y) in enumerate(zip(a, b)) if not torch.equal(x, y)]
            assert not bad, (other, e, bad[:5], len(bad))
        assert [i for i, _ in o_logs] == [i for i, _ in g_logs]
        for (i, a), (_, b) in zip(g_logs, o_logs):
            assert a == b and list(a) == list(b), (other, i)         # the same floats under the same names in the same order


def test_no_host_synchronisation_between_replays(repro, monkeypatch):
    tr = _build(CFG)
    _epochs(tr, 2, None)                                              # both graphs exist now
    counts = {"n": 0}

    def counted(obj, name):
        fn = getattr(obj, name)

        def wrapper(*a, **k):
            counts["n"] += 1
            return fn(*a, **k)
        monkeypatch.setattr(obj, name, wrapper)
    counted(torch.cuda, "synchronize")
    counted(torch.Tensor, "item")
    counted(torch.cuda.Event, "synchronize")
    counted(torch.cuda.Stream, "synchronize")
    at_replay, replay = [], torch.cuda.CUDAGraph.replay
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", lambda g: (at_replay.append(counts["n"]), replay(g))[1])
    tr.PRINT_EVERY = 3                                                # batches 0 and 3 are logged: their copies are in flight
    tr.train_one_epoch(2)
    monkeypatch.undo()
    assert len(at_replay) == 4 and at_replay[0] == at_replay[-1], at_replay


def test_checkpoint_round_trip_and_best_checkpoint(repro, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    script = [0.2, 0.1, 0.3]
    straight = _build(CFG, dropout=0.0, tester=S.StubTester(script))
    straight.train()
    best = torch.load("out/m/checkpoint_best.pth", weights_only=False)
    assert (best["epoch"], best["best_result"], best["best_epoch"]) == (3, 0.3, 3)
    assert straight.logger.lines[1::2][:3] == ["Best Result:0.2, epoch:1", "Best Result:0.2, epoch:1", "Best Result:0.3, epoch:3"]
    want = _state(straight)

    os.rename("out", "out_straight")
    first = _build(dict(CFG, max_epoch=2), dropout=0.0, tester=S.StubTester(script))
    first.train()
    saved = torch.load("out/m/checkpoint.pth", weights_only=False)
    assert (saved["epoch"], saved["best_result"], saved["best_epoch"]) == (2, 0.2, 1)
    assert len(saved["optimizer_state"]["state"]) == len(first.optimizer.bucket.params)
    assert all(s["step"] == 8 for s in saved["optimizer_state"]["state"].values())
    dev = torch.device("cuda", torch.cuda.current_device())
    seed = int(K.master_seed(dev).item())                  # the dropout seed is not part of the reference's checkpoint format
    del first
    resumed = _build(dict(CFG, resume_model=True), dropout=0.0, tester=S.StubTester(script[2:]))
    K.reseed(dev, seed)
    assert (resumed.epoch, resumed.best_result, resumed.best_epoch) == (2, 0.2, 1) and resumed.optimizer.step_count == 8
    resumed.train()
    got = _state(resumed)
    bad = [i for i, (x, y) in enumerate(zip(want, got)) if not torch.equal(x, y)]
    assert not bad, (bad[:5], len(bad))
    assert [g["lr"] for g in resumed.optimizer.param_groups] == [g["lr"] for g in straight.optimizer.param_groups]
    again = torch.load("out/m/checkpoint_best.pth", weights_only=False)
    assert (again["epoch"], again["best_result"], again["best_epoch"]) == (3, 0.3, 3)
    for k, v in best["model_state"].items():
        assert torch.equal(v, again["model_state"][k]), k
