"""CPU, gloo, world sizes 1, 2 and 3: the validation pass split over the ranks of a process group (`Tester.inference()` /
`evaluate()` / `test()`, `DeviceEvaluator.merge`, `dataset.DeviceLoader.shard`, and `Trainer.train` with a tester attached),
through the stand-in for the mdb_kitti_* entry points of tests/test_validation_host_logic.py.  Every rank must return the
AP of the single-process run, hold its merged table byte for byte, and only rank 0 may log or write files -- the same lines
and the same bytes as one process.  The split's 48 images come in batches of 5 (10 batches, the last one short), 7 (7
batches: divisible by neither 2 nor 3) and 24 (2 batches: with 3 ranks, rank 2 has none)."""
import contextlib
import io
import os
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from torch.utils.data import Dataset

import trainer_stubs as S

HERE = os.path.dirname(os.path.abspath(__file__))
BATCHES = (5, 7, 24)
WORLDS = (1, 2, 3)
THRESH = 0.95               # a few detections per image: the stand-in evaluation is a Python oracle


class _Split(Dataset):
    """The light dataset a DeviceLoader wraps: item -> (item, record), with the attributes the Tester reads."""

    def __init__(self, golden, label_dir):
        ids = golden["ids"].tolist()
        self.idx_list = ["%06d" % i for i in ids]
        self.label_dir, self.split, self.max_objs = label_dir, "val", 50
        self.writelist, self.class_name = ["Car", "Pedestrian"], ["Pedestrian", "Car", "Cyclist"]
        from oracle import decode as od
        self.cls_mean_size = od.synthetic_heads(0, 1, 1)["mean_size"]
        self.P2 = od.synthetic_heads(11, len(ids), 1)
        self.ids = ids

    def __len__(self):
        return len(self.ids)

    def __getitem__(self, item):
        return item, None


class _Bank:
    def views(self, idx):
        return list(idx)


class _Builder:
    """The batch of test_validation_host_logic's stand-in loader for split positions `idx`; records what it built."""

    def __init__(self, split):
        self.split, self.built = split, []

    def __call__(self, images, idx, records):
        self.built.append(list(idx))
        n, h = len(idx), self.split.P2
        inputs = torch.tensor(idx, dtype=torch.float32).add(1).view(n, 1, 1, 1).expand(n, 3, 4, 4).contiguous()
        info = {"img_id": torch.tensor([self.split.ids[k] for k in idx]), "img_size": torch.from_numpy(h["img_size"][idx])}
        return inputs, torch.from_numpy(h["P2"][idx]), {}, info


class _Heads(torch.nn.Module):
    """Seeded head outputs per image (seeded by its split position, so that they do not depend on the batch), with the
    depths moved by an amount set by the weight `k`, which a checkpoint sets: k = 0 gives the detections the labels lie near,
    and k = 1, 2, 3 three distinct APs."""

    def __init__(self):
        super().__init__()
        self.k = torch.nn.Parameter(torch.zeros(()))

    def forward(self, images, calibs, targets, img_sizes, dn_args=None):
        return _heads(images, int(self.k.detach()))


def _heads(images, k):
    from oracle import decode as od
    hs = [od.synthetic_heads(int(images[i, 0, 0, 0]), 1, 50) for i in range(images.shape[0])]
    h = {key: np.concatenate([x[key] for x in hs]) for key in ("logits", "boxes", "dim3", "depth", "angle")}
    h["depth"][..., 0] += np.float32(0.1 * ((2 * k) % 5))
    return {"pred_logits": torch.from_numpy(h["logits"]), "pred_boxes": torch.from_numpy(h["boxes"]),
            "pred_3d_dim": torch.from_numpy(h["dim3"]), "pred_depth": torch.from_numpy(h["depth"]),
            "pred_angle": torch.from_numpy(h["angle"])}


class _EpochHeads(_Heads):
    """`k` steps at every `eval()`, so that each validation pass of a training run sees other detections."""

    def eval(self):
        with torch.no_grad():
            self.k += 1
        return super().eval()


class _TrainedHeads(S.StubModel):
    """The stub model of the trainer tests in training mode; in eval mode the heads of `_Heads`, with `k` the number of
    training epochs so far (a buffer, so that checkpoints carry it): each validation pass of a training run sees other
    detections, and a checkpoint loaded by `Tester.test()` gives back its epoch's."""

    def __init__(self):
        super().__init__()
        self.register_buffer("k", torch.zeros(()))

    def train(self, mode=True):
        if mode:
            with torch.no_grad():
                self.k += 1
        return super().train(mode)

    def forward(self, images, calibs, targets, img_sizes, dn_args=None):
        if self.training:
            return super().forward(images, calibs, targets, img_sizes, dn_args)
        return _heads(images, int(self.k))


def _files(path):
    if not os.path.isdir(path):
        return {}
    return {f: open(os.path.join(path, f), "rb").read() for f in sorted(os.listdir(path))}


def _loader(split, batch):
    from monodetr_b200 import dataset as ds
    builder = _Builder(split)
    return ds.DeviceLoader(ds.kitti_loader(split, batch, False, 0), _Bank(), builder), builder


def _passes(split, S):
    """Tester.inference() + evaluate() per batch size: AP, log, files, merged table, the batches this rank built."""
    from monodetr_b200 import tester
    out = {}
    for batch in BATCHES:
        loader, builder = _loader(split, batch)
        log = S.ListLogger()
        t = tester.Tester({"topk": 50, "threshold": THRESH}, _Heads(), loader, log, {"save_path": f"pass{batch}"})
        t.inference()
        car = t.evaluate()
        out[batch] = {"car": car, "log": log.lines, "files": _files(f"pass{batch}/monodetr/outputs/data"),
                      "table": t.evaluator._buf.numpy().tobytes(), "built": [b[0] // batch for b in builder.built]}
    return out


def _errors(golden, H, S):
    """The add-twice and never-added errors after the merge, then a good pass on the same evaluator."""
    rank, world = (dist.get_rank(), dist.get_world_size()) if dist.is_initialized() else (0, 1)
    rows, count = torch.from_numpy(golden["rows"]), torch.from_numpy(golden["count"])
    n = len(count)
    ev = H.evaluator(golden)
    msgs = []
    for owned in ([s for s in range(n - 1) if s % world == rank],                  # the last image nowhere
                  [s for s in range(n) if s % world == rank] + [0] * (rank == world - 1)):      # image 0 twice
        ev.reset()
        if owned:
            ev.add_rows(rows[owned].clone(), count[owned].clone(), owned)
        ev.merge()
        with pytest.raises(ValueError) as e:
            ev.result(S.ListLogger())
        msgs.append(str(e.value))
        with pytest.raises(ValueError):
            ev.write_results("never_written")
    ev.reset()
    owned = [s for s in range(n) if s % world == rank]
    ev.add_rows(rows[owned].clone(), count[owned].clone(), owned)
    ev.merge()
    return msgs, ev.result(S.ListLogger()), ev._buf.numpy().tobytes(), ev.table_f.numpy().copy()


def _test_modes(S, split):
    """Tester.test() over checkpoints whose weight k is the epoch, in 'single' and 'all' mode."""
    from monodetr_b200 import tester, trainer
    out = {}
    for name, cfg in (("single", {"mode": "single", "checkpoint": 2}), ("all", {"mode": "all", "checkpoint": 2})):
        save = f"ck_{name}"
        os.makedirs(f"{save}/monodetr")
        for e in (1, 2, 3):
            m = _Heads()
            with torch.no_grad():
                m.k.fill_(e)
            trainer.save_checkpoint(trainer.get_checkpoint_state(m, None, e, 0.0, 0), f"{save}/monodetr/checkpoint_epoch_{e}")
            os.utime(f"{save}/monodetr/checkpoint_epoch_{e}.pth", (1_700_000_000 + e, 1_700_000_000 + e))
        loader, _ = _loader(split, 7)
        log = S.ListLogger()
        t = tester.Tester(dict(cfg, topk=50, threshold=THRESH), _Heads(), loader, log, {"save_path": save, "save_all": True})
        t.test()
        out[name] = {"log": log.lines,
                     "files": _files(f"{save}/monodetr/outputs/data"), "k": float(t.model.k)}
    return out


def _train(S, split):
    """Trainer.train (eager path, stub model) for 3 epochs with a Tester attached: every rank validates."""
    from monodetr_b200 import tester
    from monodetr_b200 import trainer as T
    from monodetr_b200.optim import build_lr_scheduler
    model = S.StubModel()
    opt = torch.optim.Adam(model.parameters(), lr=0.01)
    sched, warm = build_lr_scheduler(S.SCHED_CFG, opt, last_epoch=-1)
    log = S.ListLogger()
    tr = T.Trainer(dict(S.CFG, max_epoch=3, save_all=False), model, opt, S.make_loader(n_batches=3), None, sched, warm, log,
                   S.StubCriterion(), "monodetr")
    loader, _ = _loader(split, 5)
    tr.tester = tester.Tester({"topk": 50, "threshold": THRESH}, _EpochHeads(), loader, log, {"save_path": "out"})
    aps = []
    evaluate = tr.tester.evaluate

    def recording():
        aps.append(evaluate())
        return aps[-1]
    tr.tester.evaluate = recording
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        tr.train()
    best = None
    if os.path.exists("out/monodetr/checkpoint_best.pth"):
        ck = torch.load("out/monodetr/checkpoint_best.pth", weights_only=False)
        best = (ck["epoch"], ck["best_result"], ck["best_epoch"])
    # a tester that does not split its pass (the reference's) runs on rank 0 alone
    stub, model2 = S.StubTester(), S.StubModel()
    opt2 = torch.optim.Adam(model2.parameters(), lr=0.01)
    sched2, warm2 = build_lr_scheduler(S.SCHED_CFG, opt2, last_epoch=-1)
    tr2 = T.Trainer(dict(S.CFG, max_epoch=2, save_path="out_stub"), model2, opt2, S.make_loader(n_batches=2), None, sched2,
                    warm2, S.ListLogger(), S.StubCriterion(), "monodetr")
    tr2.tester = stub
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        tr2.train()
    return {"aps": aps, "log": log.lines, "ckpts": sorted(f for f in os.listdir("out/monodetr") if f.endswith(".pth"))
            if os.path.isdir("out/monodetr") else [], "files": _files("out/monodetr/outputs/data"), "best": best,
            "stub_calls": stub.calls}


def _train_then_test(split, shared, mpatch):
    """Trainer.train for 3 epochs, then Tester.test() on the same tester and model, as train_val.py runs them, in a directory
    all ranks share.  Rank 0 writes checkpoint_best.pth late: the other ranks must still load the finished file."""
    import time
    from monodetr_b200 import tester
    from monodetr_b200 import trainer as T
    from monodetr_b200.optim import build_lr_scheduler
    if not dist.is_initialized() or dist.get_rank() == 0:
        save = T.save_checkpoint

        def slow(state, filename):
            if "checkpoint_best" in filename:
                time.sleep(2)
            save(state, filename)
        mpatch.setattr(T, "save_checkpoint", slow)
    os.chdir(shared)
    model = _TrainedHeads()
    opt = torch.optim.Adam(model.parameters(), lr=0.01)
    sched, warm = build_lr_scheduler(S.SCHED_CFG, opt, last_epoch=-1)
    log = S.ListLogger()
    tr = T.Trainer(dict(S.CFG, max_epoch=3, save_all=False), model, opt, S.make_loader(n_batches=3), None, sched, warm, log,
                   S.StubCriterion(), "monodetr")
    loader, _ = _loader(split, 7)
    tr.tester = tester.Tester({"topk": 50, "threshold": THRESH, "mode": "single", "checkpoint": 0}, model, loader, log,
                              {"save_path": "out", "save_all": False})
    aps = []
    evaluate = tr.tester.evaluate

    def recording():
        aps.append(evaluate())
        return aps[-1]
    tr.tester.evaluate = recording
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        tr.train()
        tr.tester.test()
    if dist.is_initialized():
        dist.barrier()                                                 # rank 0's files are complete before any rank reads them
    return {"aps": aps, "log": log.lines, "files": _files("out/monodetr/outputs/data"), "k": float(model.k)}


def _install_fake(mpatch):
    import fake_device_lib
    import test_validation_host_logic as H
    from monodetr_b200 import _lib
    from monodetr_b200 import kitti_eval as ke
    fake_device_lib.install(mpatch)
    lib = H.ValidationFakeLib(1)
    lib.evals, lib.collects, lib.compacts = [], [], []
    mpatch.setattr(_lib, "_lib", lib)
    mpatch.setattr(ke, "_device", lambda: torch.device("cpu"))


def _write_labels(golden, label_dir):
    """Labels near the k = 0 detections of every image (as test_validation_gpu.labels_near), so that the AP is not zero."""
    from monodetr_b200 import decode
    split = _Split(golden, label_dir)
    rng = np.random.default_rng(5)
    os.makedirs(label_dir)
    for s, img_id in enumerate(split.ids):
        inputs, calibs, _, info = _Builder(split)(None, [s], None)
        dets = decode.extract_dets_from_outputs(_Heads()(inputs, calibs, None, info["img_size"]), topk=50)
        rows = decode.decode_detections(dets, {"img_id": [img_id], "img_size": info["img_size"]}, calibs,
                                        split.cls_mean_size, THRESH)[img_id]
        lines = []
        for r in rows:
            if rng.random() < 0.4:
                continue
            box = np.asarray(r[2:6]) + rng.normal(0, 2.0, 4)
            xyz = np.asarray(r[9:12]) + rng.normal(0, 0.1, 3)
            lines.append("{} 0.00 0 {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f}\n".format(
                split.class_name[int(r[0])], r[1], *box, *r[6:9], *xyz, r[12]))
        with open(os.path.join(label_dir, "%06d.txt" % img_id), "w") as f:
            f.write("".join(lines))


def _worker(rank, world, store_path, q, workdir):
    if world > 1:
        os.environ["GLOO_SOCKET_IFNAME"] = "lo"
        dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=world)
    sys.path.insert(0, HERE)
    import test_validation_host_logic as H
    mpatch = pytest.MonkeyPatch()
    _install_fake(mpatch)
    golden = dict(np.load(os.path.join(HERE, "golden", "validation.npz")))
    split = _Split(golden, os.path.join(workdir, "label_2"))
    os.chdir(os.path.join(workdir, str(world), str(rank)))
    res = {"rank": rank, "passes": _passes(split, S), "errors": _errors(golden, H, S), "test": _test_modes(S, split),
           "train": _train(S, split),
           "train_test": _train_then_test(split, os.path.join(workdir, str(world), "shared"), mpatch)}
    q.put(res)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    mpatch.undo()


@pytest.fixture(scope="module")
def runs():
    """{world: [result of rank 0, rank 1, ...]}."""
    golden = dict(np.load(os.path.join(HERE, "golden", "validation.npz")))
    tmp = tempfile.mkdtemp(prefix="mdb_gloo_validation_")
    with pytest.MonkeyPatch.context() as mpatch:
        _install_fake(mpatch)
        _write_labels(golden, os.path.join(tmp, "label_2"))
    ctx = mp.get_context("spawn")
    out = {}
    for world in WORLDS:
        for r in range(world):
            os.makedirs(os.path.join(tmp, str(world), str(r)))
        os.makedirs(os.path.join(tmp, str(world), "shared"))
        q = ctx.Queue()
        procs = [ctx.Process(target=_worker, args=(r, world, os.path.join(tmp, f"store{world}"), q, tmp)) for r in range(world)]
        for p in procs:
            p.start()
        res = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r["rank"])
        for p in procs:
            p.join(timeout=60)
            assert p.exitcode == 0
        out[world] = res
    return out


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("batch", BATCHES)
def test_pass_equals_one_process(runs, world, batch):
    one = runs[1][0]["passes"][batch]
    assert one["car"] > 0 and len(one["files"]) == 48 and one["log"][0] == "==> Saving ..."
    for r, res in enumerate(runs[world]):
        got = res["passes"][batch]
        assert got["car"] == one["car"]
        assert got["table"] == one["table"]                              # the merged table, byte for byte
        if r == 0:
            assert got["log"] == one["log"] and got["files"] == one["files"]
        else:
            assert got["log"] == [] and got["files"] == {}


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("batch", BATCHES)
def test_each_rank_builds_only_its_batches(runs, world, batch):
    n_batches = -(-48 // batch)
    for r, res in enumerate(runs[world]):
        assert res["passes"][batch]["built"] == [b for b in range(n_batches) if b % world == r]
    if world == 3 and batch == 24:
        assert runs[world][2]["passes"][batch]["built"] == []           # a rank with no work still merges


@pytest.mark.parametrize("world", WORLDS)
def test_added_twice_or_never_raises_after_the_merge(runs, world):
    one_car = float(np.load(os.path.join(HERE, "golden", "validation.npz"))["car"])
    _, _, one_table, one_f = runs[1][0]["errors"]
    assert ((one_f == 0) & np.signbit(one_f)).any()                    # the fixture holds -0.0, which a float sum would lose
    for res in runs[world]:
        (missing, twice), car, table, _ = res["errors"]
        assert "never added" in missing and "more than once" not in missing
        assert "more than once" in twice and "never added" not in twice
        assert car == one_car                                            # reset() clears what the failed passes left
        assert table == one_table                                        # merged bit for bit, -0.0 included


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("mode", ["single", "all"])
def test_tester_test_equals_one_process(runs, world, mode):
    one = runs[1][0]["test"][mode]
    assert one["k"] == (2.0 if mode == "single" else 3.0)
    assert sum(line.startswith("==> Loading from checkpoint") for line in one["log"]) == (1 if mode == "single" else 2)
    for r, res in enumerate(runs[world]):
        got = res["test"][mode]
        assert got["k"] == one["k"]
        if r == 0:
            assert got["log"] == one["log"] and got["files"] == one["files"]
        else:
            assert got["log"] == [] and got["files"] == {}


@pytest.mark.parametrize("world", [2, 3])
def test_trainer_validates_on_every_rank(runs, world):
    one = runs[1][0]["train"]
    assert one["aps"][2] > one["aps"][0] > one["aps"][1]          # epoch 1 is the best until epoch 3 beats it
    assert one["ckpts"] == ["checkpoint.pth", "checkpoint_best.pth"]
    best = max(range(3), key=lambda e: one["aps"][e])
    assert one["best"] == (best + 1, one["aps"][best], best + 1)
    assert one["log"][-1] == "Best Result:{}, epoch:{}".format(one["aps"][best], best + 1)
    for r, res in enumerate(runs[world]):
        got = res["train"]
        assert got["aps"] == one["aps"]
        if r == 0:
            assert got["log"] == one["log"] and got["files"] == one["files"] and got["best"] == one["best"]
            assert got["ckpts"] == one["ckpts"]
        else:
            assert got["log"] == [] and got["files"] == {} and got["ckpts"] == [] and got["best"] is None
    assert one["stub_calls"] == 2
    for r, res in enumerate(runs[world]):
        assert res["train"]["stub_calls"] == (2 if r == 0 else 0)


@pytest.mark.parametrize("world", [2, 3])
def test_train_then_test_loads_the_finished_best_checkpoint(runs, world):
    one = runs[1][0]["train_test"]
    assert one["aps"][2] > one["aps"][0] > one["aps"][1]          # the last epoch writes a new checkpoint_best.pth
    assert one["aps"][3] == one["aps"][2] and one["k"] == 3.0      # test() evaluates it
    assert len(one["files"]) == 48
    for r, res in enumerate(runs[world]):
        got = res["train_test"]
        assert got["aps"] == one["aps"] and got["k"] == one["k"]
        assert got["files"] == one["files"]                              # the directory all ranks share
        assert got["log"] == (one["log"] if r == 0 else [])
