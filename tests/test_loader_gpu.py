"""GPU: monodetr_b200.dataset.build_dataloader against the reference loader (tests/golden/loader.npz, tools/gen_golden_loader.py)
on the same synthetic KITTI folder (tests/synthetic_kitti.py): every recorded batch of the train loader (0 and 2 workers, two
epochs), the val loader and the test loader -- `inputs` bit-identical, `calibs` and `info` exact, targets within the label
encoder's bounds (oracle.labels.assert_targets_match); the image banks against PIL; and, in reproducible mode, a Trainer epoch
on the graph path and a Tester pass fed by the new loaders against the same fed by host-decoded images through
KittiBatchBuilder with the same records."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch
from PIL import Image

import monodetr_b200
import synthetic_kitti as sk
import trainer_stubs as S
from monodetr_b200 import dataset as ds
from oracle import labels as ol

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "loader.npz"))
CFG = json.loads(str(GOLD["cfg"]))
RUNS = {"train_w0": ("val", 0, 2), "train_w2": ("val", 2, 2), "val": ("val", 0, 1), "test": ("test", 0, 1)}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    sk.write_tree(root)
    return root


def _cfg(root, **over):
    return dict(CFG, root_dir=root, **over)


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("split", ["train", "val", "test"])
def test_bank_bytes_equal_the_pil_decode(tree, split):
    bank = ds.ImageBank(tree, split, threads=3)
    data = os.path.join(tree, "testing" if split == "test" else "training")
    assert len(bank) == len(GOLD[f"tree.sha.{split}"])
    for k, (img_id, v) in enumerate(zip(bank.img_ids, bank.views(range(len(bank))))):
        want = np.array(Image.open(os.path.join(data, "image_2", "%06d.png" % img_id)))
        got = v.cpu().numpy()
        assert v.is_cuda and got.shape == want.shape and v.data_ptr() == bank.data.data_ptr() + int(bank.offsets[k])
        assert np.array_equal(got, want) and _sha(got) == str(GOLD[f"tree.sha.{split}"][k])


@pytest.mark.parametrize("run", list(RUNS))
def test_batches_match_the_reference_loader(tree, run):
    test_split, workers, epochs = RUNS[run]
    sk.set_random_seed(444)
    train_loader, test_loader = ds.build_dataloader(_cfg(tree, test_split=test_split), workers=workers)
    loader = train_loader if run.startswith("train") else test_loader
    for epoch in range(epochs):
        if loader is train_loader:
            np.random.seed(np.random.get_state()[1][0] + epoch)          # Trainer.train, before each epoch
        p = f"{run}.e{epoch}"
        bounds = GOLD[p + ".bounds"]
        assert len(loader) == len(bounds) - 1
        n = 0
        for b, (inputs, calibs, targets, info) in enumerate(loader):
            lo, hi = int(bounds[b]), int(bounds[b + 1])
            assert inputs.is_cuda and calibs.is_cuda and not info["img_id"].is_cuda and inputs.shape == (hi - lo, 3, 384, 1280)
            x = inputs.cpu().numpy()
            for i in range(hi - lo):
                assert _sha(x[i]) == str(GOLD[p + ".sha"][lo + i]), (p, b, i)
                np.testing.assert_array_equal(x[i].reshape(-1)[GOLD[p + ".sample_pos"][lo + i]], GOLD[p + ".sample_val"][lo + i])
            np.testing.assert_array_equal(calibs.cpu().numpy(), GOLD[p + ".calibs"][lo:hi])
            assert calibs.dtype == torch.float32
            for k, key in (("img_id", "info_img_id"), ("img_size", "info_img_size"), ("bbox_downsample_ratio", "info_ratio")):
                assert info[k].dtype == torch.from_numpy(GOLD[p + "." + key]).dtype, k
                np.testing.assert_array_equal(info[k].numpy(), GOLD[p + "." + key][lo:hi], err_msg=k)
            if run == "test":
                assert targets is inputs
            else:
                got = {k: v.cpu().numpy() for k, v in targets.items()}
                ol.assert_targets_match(got, {k: GOLD[f"{p}.t.{k}"][lo:hi] for k in ol.KEYS}, f"{p} batch {b}")
                for k in ol.KEYS + ("img_size",):
                    assert got[k].dtype == GOLD[f"{p}.t.{k}"].dtype, k
                np.testing.assert_array_equal(got["img_size"], GOLD[f"{p}.t.img_size"][lo:hi])
            n += hi - lo
        assert n == int(bounds[-1])


# ---- end to end: Trainer and Tester fed by the device loader vs host-decoded images ------------------------------------------
class _HostDecoded:
    """Today's route: each batch's images decoded by PIL in the main process and handed over as CPU tensors."""

    def __init__(self, root, split):
        self.dir = os.path.join(root, "training", "image_2")
        self.ids = [int(x) for x in open(os.path.join(root, "ImageSets", split + ".txt"))]

    def views(self, idx):
        return [torch.from_numpy(np.array(Image.open(os.path.join(self.dir, "%06d.png" % self.ids[k])))) for k in idx]


def _loaders(root, device_route):
    from monodetr_b200.labels import KittiBatchBuilder, LabelBank
    cfg = _cfg(root)
    if device_route:
        return ds.build_dataloader(cfg, workers=2)
    out = []
    for split, shuffle in ((cfg["train_split"], True), (cfg["test_split"], False)):
        dataset = ds.KITTI_Dataset(split, cfg)
        builder = KittiBatchBuilder(cfg, split, LabelBank.from_kitti(root, split))
        out.append(ds.DeviceLoader(ds.kitti_loader(dataset, cfg["batch_size"], shuffle, 2), _HostDecoded(root, split), builder))
    return out


def _run(root, out_dir, device_route):
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr, kernels as K, tc
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    from monodetr_b200.tester import Tester
    from monodetr_b200.trainer import Trainer
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG))
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler({"warmup": False, "decay_rate": 0.5, "decay_list": [1]}, opt, last_epoch=-1)
    sk.set_random_seed(444)
    train_loader, val_loader = _loaders(root, device_route)
    tr = Trainer({"max_epoch": 1, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": out_dir}, model, opt,
                 train_loader, val_loader, sched, warm, S.ListLogger(), crit, "m")
    assert tr.graph_path
    K.reseed(torch.device("cuda", torch.cuda.current_device()), 4242)
    np.random.seed(np.random.get_state()[1][0] + 0)
    tr.train_one_epoch(0)
    assert tr.live_graphs == 1                                    # batch 0 eager, 1-2 replayed, the short last one eager
    params = [p.detach().clone() for p in model.parameters()] + [opt.exp_avg.clone(), opt.exp_avg_sq.clone()]
    log = S.ListLogger()
    tester = Tester({"topk": 50, "threshold": 0.0}, model, val_loader, log, {"save_path": out_dir}, "m")
    was = torch.is_grad_enabled()
    try:
        tester.inference()
    finally:
        torch.set_grad_enabled(was)
    ap = tester.evaluate()
    res = os.path.join(out_dir, "m", "outputs", "data")
    files = {f: open(os.path.join(res, f)).read() for f in sorted(os.listdir(res))}
    return params, files, ap, log.lines


def test_trainer_and_tester_match_the_host_decoded_route(tree, tmp_path, monkeypatch):
    from monodetr_b200 import trainer as T
    monkeypatch.setattr(T, "print_losses", lambda i, log: None)
    monkeypatch.chdir(tmp_path)
    prev = monodetr_b200.set_deterministic(True)
    try:
        new = _run(tree, "new", True)
        old = _run(tree, "old", False)
    finally:
        monodetr_b200.set_deterministic(prev)
    bad = [i for i, (a, b) in enumerate(zip(new[0], old[0])) if not torch.equal(a, b)]
    assert len(new[0]) == len(old[0]) and not bad, bad[:5]
    assert new[1] == old[1] and len(new[1]) == 6 and any(new[1].values())
    assert new[2] == old[2] and new[3] == old[3]
