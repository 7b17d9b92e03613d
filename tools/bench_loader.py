"""What the KITTI loader costs: monodetr_b200.dataset.build_dataloader (device image and label banks) against a CPU loader built
the way the reference's works (per item: PIL decode, photometric distortion, flip, warp, normalisation and label encoding in numpy
on loader workers -- here the repository's oracle restatements oracle/photometric.py, oracle/preprocess.py, oracle/labels.py
stand in for the reference's code), on a synthetic KITTI folder (tests/synthetic_kitti.py) with the shipped dataset section.

    python tools/bench_loader.py [--train 256] [--val 64] [--batch 16] [--out FILE]

Prints one JSON line (and writes it to --out) with the GPU's name and power limit read in the same run:
  bank_build_s             ImageBank of the train split by decode thread count (host clock, ends in a synchronise)
  assembly_ms              one batch through KittiBatchBuilder from bank views: device events around the call, and the host
                           clock around call + synchronise (median and max over the timed batches)
  loader_batches_per_s     one epoch of each loader iterated with nothing else, the device loader ending in a synchronise
  trainer_epoch_s          Trainer.train_one_epoch on the graph path fed by each loader (model, device criterion, FusedAdamW)
  peak_device_bytes        torch.cuda.max_memory_allocated over the train and val banks, their label banks and the first
                           training epoch at the batch size (which includes the captured graph's memory)
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHIPPED = {"type": "KITTI", "train_split": "train", "test_split": "val", "use_3d_center": True, "class_merging": False,
           "use_dontcare": False, "bbox2d_type": "anno", "meanshape": False, "writelist": ["Car"], "clip_2d": False, "aug_pd": True,
           "aug_crop": True, "random_flip": 0.5, "random_crop": 0.5, "scale": 0.05, "shift": 0.05, "depth_scale": "normal"}


class OracleDataset(torch.utils.data.Dataset):
    """kitti_dataset.py's __getitem__ on the host, per item, from the oracle restatements."""

    def __init__(self, split, cfg):
        from monodetr_b200 import dataset as ds
        self.light = ds.KITTI_Dataset(split, cfg)

    def __len__(self):
        return len(self.light)

    def __getitem__(self, item):
        from PIL import Image
        from monodetr_b200.labels import parse_calib_file, parse_label_file
        from oracle import labels as ol, photometric as oph, preprocess as opp
        d = self.light
        img_id = int(d.idx_list[item])
        img = np.array(Image.open(os.path.join(d.image_dir, "%06d.png" % img_id)))
        _, rec = d[item]
        if rec.distort is not None:
            img = oph.distort(img, oph.Params(*rec.distort))
        inputs = opp.preprocess(img, np.asarray(rec.trans_inv).reshape(6), tuple(d.resolution), rec.flip)
        P2 = parse_calib_file(os.path.join(d.calib_dir, "%06d.txt" % img_id))
        _, objs = parse_label_file(os.path.join(d.label_dir, "%06d.txt" % img_id))
        t = ol.encode_image(objs, P2, rec.img_size, rec.flip, rec.crop_scale, rec.trans)
        targets = {k: v[0] for k, v in t.items()}
        targets["img_size"] = np.array(rec.img_size)
        size = np.array(rec.img_size)
        info = {"img_id": img_id, "img_size": size, "bbox_downsample_ratio": size / (d.resolution // 32)}
        return inputs, P2, targets, info


def oracle_loader(cfg, split, shuffle, workers):
    from monodetr_b200.dataset import my_worker_init_fn
    return torch.utils.data.DataLoader(OracleDataset(split, cfg), batch_size=cfg["batch_size"], num_workers=workers,
                                       worker_init_fn=my_worker_init_fn, shuffle=shuffle, pin_memory=False, drop_last=False)


class _Logger:
    def info(self, msg):
        pass


def build_trainer(loader):
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    from monodetr_b200.trainer import Trainer
    torch.manual_seed(0)
    model, _ = build_monodetr(DEFAULT_MODEL_CFG)
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler({"warmup": True, "decay_rate": 0.1, "decay_list": [125, 165]}, opt, last_epoch=-1)
    cfg = {"max_epoch": 1, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": "unused"}
    tr = Trainer(cfg, model, opt, loader, None, sched, warm, _Logger(), crit, "bench")
    assert tr.graph_path
    return tr


def timed_epoch(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def drain(loader):
    for _ in loader:
        pass


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train", type=int, default=256)
    ap.add_argument("--val", type=int, default=64)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--threads", type=int, nargs="+", default=[1, 4, 8, 16])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loader: a CUDA device is required (nothing is measured without one)")
    import synthetic_kitti as sk
    from monodetr_b200 import dataset as ds
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "batch": args.batch, "train_images": args.train, "val_images": args.val, "resolution": "1280x384",
           "host_cpus": os.cpu_count()}
    with tempfile.TemporaryDirectory() as root:
        t0 = time.perf_counter()
        sk.write_tree(root, n_train=args.train, n_val=args.val, n_test=1, seed=1)
        res["tree_write_s"] = round(time.perf_counter() - t0, 1)
        cfg = dict(SHIPPED, root_dir=root, batch_size=args.batch)
        sk.set_random_seed(444)

        # banks + the first training epoch: peak device memory; the graph is captured in this epoch
        torch.cuda.reset_peak_memory_stats()
        train_dev, val_dev = ds.build_dataloader(cfg, workers=4)
        res["bank_bytes"] = {"train": int(train_dev.bank.data.numel()), "val": int(val_dev.bank.data.numel())}
        tr = build_trainer(train_dev)
        res["trainer_warm_epoch_s"] = round(timed_epoch(lambda: tr.train_one_epoch(0)), 2)
        res["peak_device_bytes"] = int(torch.cuda.max_memory_allocated())

        # Trainer epochs fed by each loader (same trainer, same batch shape: every batch replays the captured graph)
        cpu4 = oracle_loader(cfg, "train", True, 4)
        ep = {"device_loader_w4": [], "cpu_oracle_loader_w4": []}
        for _ in range(2):
            tr.train_loader = train_dev
            ep["device_loader_w4"].append(round(timed_epoch(lambda: tr.train_one_epoch(1)), 3))
        tr.train_loader = cpu4
        ep["cpu_oracle_loader_w4"].append(round(timed_epoch(lambda: tr.train_one_epoch(1)), 3))
        res["trainer_epoch_s"] = ep
        res["trainer_batches_per_epoch"] = len(train_dev)

        # the loaders alone
        rate = {}
        for w in (0, 4):
            loader = ds.DeviceLoader(ds.kitti_loader(train_dev.dataset, args.batch, True, w), train_dev.bank, train_dev.builder)
            drain(loader)
            rate[f"device_w{w}"] = [round(len(loader) / timed_epoch(lambda: drain(loader)), 2) for _ in range(2)]
        t0 = time.perf_counter()
        drain(cpu4)
        rate["cpu_oracle_w4"] = [round(len(cpu4) / (time.perf_counter() - t0), 3)]
        res["loader_batches_per_s"] = rate

        # one batch's assembly from bank views (records drawn beforehand)
        d = train_dev.dataset
        g = np.random.default_rng(0)
        batches = [g.permutation(len(d))[:args.batch].tolist() for _ in range(33)]
        recs = [[d[k][1] for k in idx] for idx in batches]
        dev_ms, host_ms = [], []
        for i, (idx, rr) in enumerate(zip(batches, recs)):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            train_dev.builder(train_dev.bank.views(idx), idx, rr)
            e1.record()
            torch.cuda.synchronize()
            if i >= 3:
                host_ms.append((time.perf_counter() - t0) * 1e3)
                dev_ms.append(e0.elapsed_time(e1))
        res["assembly_ms"] = {"device_events_median": round(float(np.median(dev_ms)), 3), "device_events_max": round(max(dev_ms), 3),
                              "host_clock_median": round(float(np.median(host_ms)), 3), "host_clock_max": round(max(host_ms), 3),
                              "batches": len(dev_ms)}

        # bank build by decode threads
        del tr, train_dev, val_dev
        torch.cuda.empty_cache()
        build = {}
        for t in args.threads:
            times = []
            for _ in range(2):
                t0 = time.perf_counter()
                bank = ds.ImageBank(root, "train", threads=t)
                times.append(round(time.perf_counter() - t0, 3))
                del bank
                torch.cuda.empty_cache()
            build[str(t)] = times
        res["bank_build_s"] = build
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
