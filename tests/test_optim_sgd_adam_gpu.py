"""GPU: `FusedSGD` / `FusedAdam` (csrc/optim.cu `mdb_sgd_*` / `mdb_adam_*`, monodetr_b200/optim.py) against torch.optim.SGD /
torch.optim.Adam stepping on the SAME device with the same gradients -- torch's multi-tensor (`foreach`) kernels, which is what
the reference runs -- and the `Trainer` replaying either one inside its CUDA graph on the real model.

Bound.  The kernels repeat torch's per-element operations in torch's order, with an explicit fmaf exactly where torch's kernels
contract (DeviceAddCmulCdiv.cuh, Lerp.h, the alpha forms of `_foreach_add`), and take the same fp32 roundings of torch's fp64
step scalars, so the expected difference is zero.  What can differ is the fp64 `pow` in the bias corrections of Adam's
device-side step scalars (CUDA's against the host's libm), by one fp64 ulp, which moves the fp32 rounding of a scalar by at most
one ulp in rare cases; that scales an update by 2^-23 relative.  rtol 4e-7 (about 3 ulp) on parameters and state after six steps
covers that with room and fails for any change of operation order that matters (a dropped FMA moves single elements by up to
1 ulp per step, a wrong lerp branch or bias correction by far more).  Whether the run was bit-exact is printed."""
import copy
import os

import pytest
import torch

import monodetr_b200
import trainer_stubs as S
from monodetr_b200 import kernels as K

pytestmark = pytest.mark.gpu

KINDS = ("sgd", "adam")
RTOL, ATOL = 4e-7, 1e-12


@pytest.fixture
def repro():
    prev = monodetr_b200.set_deterministic(True)
    try:
        yield
    finally:
        monodetr_b200.set_deterministic(prev)


def _toy(seed=0):
    torch.manual_seed(seed)
    return torch.nn.ModuleDict({
        "a": torch.nn.Linear(37, 19),            # odd sizes: alignment padding between the tensors of the flat buffer
        "norm": torch.nn.LayerNorm(19),
        "sa_v_proj": torch.nn.Linear(3, 3),      # a name the bucket leaves out: never receives a gradient
        "b": torch.nn.Linear(19, 3),
        "emb": torch.nn.Embedding(11, 5),
    }).cuda()


def _reference(kind, model, lr, wd):
    """lib/helpers/optimizer_helper.py:7-27: all named parameters, biases (no decay) then weights."""
    named = list(model.named_parameters())
    groups = [{"params": [p for n, p in named if "bias" in n], "weight_decay": 0},
              {"params": [p for n, p in named if "bias" not in n], "weight_decay": wd}]
    return torch.optim.SGD(groups, lr=lr, momentum=0.9) if kind == "sgd" else torch.optim.Adam(groups, lr=lr)


def _fused(kind, model, lr, wd, device_step):
    from monodetr_b200.optim import FusedAdam, FusedSGD
    cls = FusedSGD if kind == "sgd" else FusedAdam
    return cls(model, lr=lr, weight_decay=wd, device_step=device_step)


class _Pair:
    """A fused optimizer and torch's over two copies of one model, fed the same gradients."""

    def __init__(self, kind, device_step, lr=2e-3, wd=1e-2):
        self.model = _toy()
        self.ref_model = copy.deepcopy(self.model)
        self.before = {n: p.detach().clone() for n, p in self.model.named_parameters()}
        self.opt = _fused(kind, self.model, lr, wd, device_step)
        self.ref = _reference(kind, self.ref_model, lr, wd)
        self.names = self.opt.bucket.names
        self.ref_params = dict(self.ref_model.named_parameters())
        self.gen = torch.Generator(device="cuda").manual_seed(1)
        self.steps = 0

    def grads(self):
        self.steps += 1
        gs = [torch.randn(p.shape, device="cuda", generator=self.gen) * (0.5 + self.steps) for p in self.opt.bucket.params]
        for p, n, g in zip(self.opt.bucket.params, self.names, gs):
            p.grad = g.clone()
            self.ref_params[n].grad = g.clone()

    def step_ref(self):
        self.ref.step()

    def compare(self, what):
        exact = True
        for n, p in zip(self.names, self.opt.bucket.params):
            r = self.ref_params[n].detach()
            assert torch.allclose(p.detach(), r, rtol=RTOL, atol=ATOL), (what, n, float((p.detach() - r).abs().max()))
            exact = exact and torch.equal(p.detach(), r)
            st, off = self.ref.state[self.ref_params[n]], self.opt.bucket.offsets[self.names.index(n)]
            for s in self.opt.STATE:
                mine = getattr(self.opt, s)[off:off + p.numel()].view_as(p)
                assert torch.allclose(mine, st[s], rtol=RTOL, atol=ATOL), (what, n, s)
                exact = exact and torch.equal(mine, st[s])
        return exact


def _untouched(pair):
    b, opt = pair.opt.bucket, pair.opt
    used = torch.zeros(b.numel, dtype=torch.bool, device="cuda")
    for off, p in zip(b.offsets, b.params):
        used[off:off + p.numel()] = True
    for s in ("flat_p",) + opt.STATE:
        assert not getattr(opt, s)[~used].any(), s                                          # padding stays zero
    for n in ("sa_v_proj.weight", "sa_v_proj.bias"):
        assert torch.equal(dict(pair.model.named_parameters())[n], pair.before[n]), n       # no gradient: untouched


@pytest.mark.parametrize("device_step", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_fused_step_matches_torch(kind, device_step):
    pair = _Pair(kind, device_step)
    b = pair.opt.bucket
    assert b.n_decay == b.offsets[b.names.index("a.bias")] and all(p.data_ptr() % 128 == 0 for p in b.params)
    exact = True
    for step in range(6):
        pair.grads()
        pair.opt.step()
        pair.step_ref()
        exact = pair.compare(step) and exact
    assert pair.opt.step_count == 6
    _untouched(pair)
    print(kind, "device_step" if device_step else "eager", "bit-exact vs torch.optim (foreach):", exact)


@pytest.mark.parametrize("kind", KINDS)
def test_schedule_and_first_step_reach_a_replayed_graph(kind):
    """Captured before any step: the first replay is torch's first step (SGD: buf = d), decided on the device; a learning rate
    `build_lr_scheduler` changes between replays is what the next replay uses."""
    from monodetr_b200.optim import build_lr_scheduler
    sched_cfg = {"warmup": False, "decay_rate": 0.25, "decay_list": [2]}
    pair = _Pair(kind, True)
    graph_grads = [torch.zeros_like(p) for p in pair.opt.bucket.params]
    for p, g in zip(pair.opt.bucket.params, graph_grads):
        p.grad = g
    sched, _ = build_lr_scheduler(sched_cfg, pair.opt, last_epoch=-1)
    ref_sched, _ = build_lr_scheduler(sched_cfg, pair.ref, last_epoch=-1)
    pair.opt.sync_hyper()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        pair.opt.step()
    assert pair.opt.step_count == 0                                         # capturing executed nothing
    for step in range(4):
        pair.grads()
        for p, g in zip(pair.opt.bucket.params, graph_grads):
            g.copy_(p.grad)
            p.grad = g
        graph.replay()
        pair.step_ref()
        pair.compare(step)
        sched.step()
        ref_sched.step()
        pair.opt.sync_hyper()
    assert pair.opt.step_count == 4 and pair.opt.param_groups[0]["lr"] == pair.ref.param_groups[0]["lr"] == 2e-3 * 0.25
    _untouched(pair)


def test_adam_device_scalars_equal_the_host_values():
    import numpy as np
    from monodetr_b200 import _lib
    pair = _Pair("adam", True, lr=2e-4)
    ts = list(range(1, 2001)) + [4999, 10 ** 4, 123457, 10 ** 6, 5 * 10 ** 6]
    out = torch.zeros(len(ts), 2, device="cuda")
    for i, t in enumerate(ts):
        if t > 2000:
            pair.opt.step_count = t - 1
        _lib.call("mdb_adam_advance", pair.opt._hyper)
        out[i].copy_(pair.opt._scalars)
    host = np.array([[np.float32((2e-4 / (1 - 0.9 ** float(t))) * -1), np.float32((1 - 0.999 ** float(t)) ** 0.5)] for t in ts])
    got = out.cpu().numpy()
    bad = [(t, list(h), list(g)) for t, h, g in zip(ts, host, got) if (h != g).any()]
    assert not bad, bad[:10]


@pytest.mark.parametrize("device_step", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_state_dict_equals_torch_and_torch_state_continues(kind, device_step):
    for taken in (3, 0):
        pair = _Pair(kind, device_step)
        for _ in range(taken):
            pair.grads()
            pair.opt.step()
            pair.step_ref()
        sd, ref_sd = pair.opt.state_dict(), pair.ref.state_dict()
        assert sd["param_groups"] == ref_sd["param_groups"] and list(sd["state"]) == list(ref_sd["state"])
        named = [n for n, _ in pair.model.named_parameters()]
        order = [n for n in named if "bias" in n] + [n for n in named if "bias" not in n]          # the reference's numbering
        assert sorted(order[i] for i in sd["state"]) == (sorted(pair.names) if taken else [])
        for i, s in ref_sd["state"].items():
            assert list(sd["state"][i]) == list(s)
            for k, v in s.items():
                if k == "step":
                    assert sd["state"][i][k].dtype == v.dtype == torch.float32 and float(sd["state"][i][k]) == float(v) == taken
                else:
                    assert torch.allclose(sd["state"][i][k], v, rtol=RTOL, atol=ATOL), (i, k)
        # torch's state -> a fresh fused optimizer over torch's parameters -> both continue on the same trajectory
        fresh = _Pair(kind, device_step)
        with torch.no_grad():
            for (n, p), (_, q) in zip(fresh.model.named_parameters(), pair.ref_model.named_parameters()):
                p.copy_(q)
                fresh.ref_params[n].copy_(q)
        fresh.opt.load_state_dict(ref_sd)
        fresh.ref.load_state_dict(ref_sd)
        fresh.gen.manual_seed(7)
        for step in range(3):
            fresh.grads()
            fresh.opt.step()
            fresh.step_ref()
            fresh.compare((taken, step))


# ---- the trainer on the real model ----------------------------------------------------------------------------------------------
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


def _build(kind, cfg, dropout=0.1, env_no_graph=False, max_graphs=None, tester=None):
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr, tc
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import build_lr_scheduler
    from monodetr_b200.trainer import Trainer
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, dropout=dropout))
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    crit.depth_map_scale = (W // 16, H // 16)
    opt = _fused(kind, model, 2e-4, 1e-4, True)
    sched, warm = build_lr_scheduler(SCHED, opt, last_epoch=-1)
    if env_no_graph:
        os.environ["MDB_NO_GRAPH"] = "1"
    try:
        tr = Trainer(cfg, model, opt, _loader(), None, sched, warm, S.ListLogger(), crit, "m")
    finally:
        os.environ.pop("MDB_NO_GRAPH", None)
    if max_graphs is not None:
        tr.MAX_GRAPHS = max_graphs
    tr.tester = tester
    K.reseed(torch.device("cuda", torch.cuda.current_device()), 4242)
    return tr


def _state(tr):
    opt = tr.optimizer
    return [opt.flat_p.clone()] + [getattr(opt, s).clone() for s in opt.STATE] + [torch.tensor(float(opt.step_count))] + \
        [p.detach().clone() for p in tr.model.parameters()]


def _epochs(tr, n):
    states = []
    for epoch in range(n):
        tr.train_one_epoch(epoch)
        tr.epoch += 1
        tr.lr_scheduler.step()
        tr.optimizer.sync_hyper()
        states.append(_state(tr))
    return states


def _same(a, b):
    return [i for i, (x, y) in enumerate(zip(a, b)) if not torch.equal(x, y)]


@pytest.mark.parametrize("kind", KINDS)
def test_trainer_graph_path_equals_eager_path(kind, repro, monkeypatch):
    from monodetr_b200 import trainer as T
    monkeypatch.setattr(T, "print_losses", lambda i, log: None)
    runs = {}
    for name, kw in (("graph", {}), ("graph_again", {}), ("eager_device_step", {"max_graphs": 0}),
                     ("reference_loop", {"env_no_graph": True})):
        tr = _build(kind, CFG, **kw)
        assert tr.graph_path == (name != "reference_loop")
        runs[name] = _epochs(tr, 3)
        if name.startswith("graph"):
            assert tr.live_graphs == 2
        assert tr.optimizer.step_count == 12
    for other in ("graph_again", "eager_device_step", "reference_loop"):
        for e, (a, b) in enumerate(zip(runs["graph"], runs[other])):
            bad = _same(a, b)
            assert not bad, (kind, other, e, bad[:5], len(bad))
    assert _same(runs["graph"][0], runs["graph"][-1])                           # it trained


@pytest.mark.parametrize("kind", KINDS)
def test_trainer_checkpoint_resumes(kind, repro, tmp_path, monkeypatch):
    from monodetr_b200 import trainer as T
    monkeypatch.setattr(T, "print_losses", lambda i, log: None)
    monkeypatch.chdir(tmp_path)
    straight = _build(kind, CFG, dropout=0.0)
    straight.train()
    want = _state(straight)
    os.rename("out", "out_straight")
    first = _build(kind, dict(CFG, max_epoch=2), dropout=0.0)
    first.train()
    saved = torch.load("out/m/checkpoint.pth", weights_only=False)["optimizer_state"]
    assert len(saved["state"]) == len(first.optimizer.bucket.params)
    assert all(list(s) == (["momentum_buffer"] if kind == "sgd" else ["step", "exp_avg", "exp_avg_sq"]) for s in saved["state"].values())
    ref = _reference(kind, first.model, 1.0, 1e-4)
    ref.load_state_dict(saved)                                                    # torch's optimizer reads the file
    dev = torch.device("cuda", torch.cuda.current_device())
    seed = int(K.master_seed(dev).item())
    del first
    resumed = _build(kind, dict(CFG, resume_model=True), dropout=0.0)
    K.reseed(dev, seed)
    assert resumed.epoch == 2 and resumed.optimizer.step_count == (1 if kind == "sgd" else 8)
    resumed.train()
    got = _state(resumed)
    n_count = 1 + len(resumed.optimizer.STATE)                                    # the step counts differ for SGD by design
    bad = [i for i in _same(want, got) if not (kind == "sgd" and i == n_count)]
    assert not bad, (bad[:5], len(bad))
