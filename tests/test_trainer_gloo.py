"""CPU, world_size 2, gloo: `trainer.Trainer` on its eager path with the stub model and criterion of tests/trainer_stubs.py -- the
ranks see different batches, end with equal parameters, log the mean over ranks, and only rank 0 writes files."""
import contextlib
import io
import os
import tempfile

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _worker(rank, world, store_path, q, workdir):
    os.environ["GLOO_SOCKET_IFNAME"] = "lo"
    dist.init_process_group("gloo", init_method=f"file://{store_path}", rank=rank, world_size=world)
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import trainer_stubs as S
    from monodetr_b200 import trainer as T
    from monodetr_b200.optim import build_lr_scheduler
    os.chdir(os.path.join(workdir, str(rank)))
    model = S.StubModel()
    with torch.no_grad():
        for p in model.parameters():
            p.add_(float(rank))                    # the constructor's broadcast must equalise
    named = list(model.named_parameters())
    opt = torch.optim.Adam([{"params": [p for n, p in named if "bias" in n], "weight_decay": 0},
                            {"params": [p for n, p in named if "bias" not in n], "weight_decay": 0.01}], lr=0.01)
    sched, warm = build_lr_scheduler(S.SCHED_CFG, opt, last_epoch=-1)
    logs = []
    T.print_losses = lambda i, log: logs.append((i, dict(log)))
    tr = T.Trainer(dict(S.CFG, max_epoch=2), model, opt, S.make_loader(n_batches=4), None, sched, warm, S.ListLogger(), S.StubCriterion(), "stub")
    tr.PRINT_EVERY = 1
    own = []                                       # this rank's un-reduced terms of every batch
    crit_forward = tr.detr_loss.forward

    def recording(outputs, targets, mask_dict=None):
        d = crit_forward(outputs, targets, mask_dict)
        own.append({k: float(v.detach() * S.StubCriterion.weight_dict[k]) for k, v in d.items() if k in S.StubCriterion.weight_dict})
        return d
    tr.detr_loss.forward = recording
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        tr.train()
    files = sorted(os.listdir("out/stub")) if os.path.isdir("out/stub") else []
    q.put((rank, [p.detach().tolist() for p in model.parameters()], tr.last_log, own[-1], len(logs), files))
    dist.barrier()
    dist.destroy_process_group()


def test_trainer_eager_path_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    tmp = tempfile.mkdtemp(prefix="mdb_gloo_trainer_")
    for r in range(2):
        os.makedirs(os.path.join(tmp, str(r)))
    procs = [ctx.Process(target=_worker, args=(r, 2, os.path.join(tmp, "store"), q, tmp)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted([q.get(timeout=600) for _ in procs], key=lambda r: r[0])
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, p0, log0, own0, n0, files0), (_, p1, log1, own1, n1, files1) = res
    assert p0 == p1
    assert files0 == ["checkpoint_epoch_1.pth", "checkpoint_epoch_2.pth"] and files1 == []
    assert n0 == 8 and n1 == 0                                         # only rank 0 prints
    assert log0 == log1 and list(log0) == sorted(own0) + ["loss_detr"]   # misc.reduce_dict: keys in sorted order
    assert own0 != own1
    for k in own0:
        assert abs(log0[k] - (own0[k] + own1[k]) / 2) < 1e-5, k
