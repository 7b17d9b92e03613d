"""Wall time of one validation pass (`Tester.inference()` + `evaluate()`) at world sizes 1, 2 and 8, one process per GPU, over a
val-sized synthetic KITTI split (tests/synthetic_kitti.py: 64 distinct images, hard-linked under 3769 ids), and of one `Trainer` epoch with that tester attached (graph path,
default model with random weights, device criterion, `FusedAdamW`).

    python tools/bench_dist_validation.py [--val 3769] [--train 256] [--batch 32] [--train-batch 8] [--worlds 1 2 8]

Each world size runs under torchrun (`--standalone`) with the loaders of `build_dataloader` on every rank.  A pass is timed with
the host clock from a barrier to a barrier after `evaluate()` returned, all ranks synchronised with the device; the first pass
warms every shape and is not counted.  A world size larger than the visible GPU count is reported as "not measured".  Prints
one JSON line with the GPU's name and power limit, read in the same run.  The synthetic tree is written to a temporary
directory."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

DATASET = {"type": "KITTI", "train_split": "train", "test_split": "val", "use_3d_center": True, "class_merging": False,
           "use_dontcare": False, "bbox2d_type": "anno", "meanshape": False, "writelist": ["Car"], "clip_2d": False,
           "aug_pd": True, "aug_crop": True, "random_flip": 0.5, "random_crop": 0.5, "scale": 0.05, "shift": 0.05,
           "depth_scale": "normal"}


class _Quiet:
    def info(self, msg):
        pass


def _sync_barrier(world):
    torch.cuda.synchronize()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()


def worker(a):
    """One rank: build the loaders, time `--repeats` validation passes and one Trainer epoch with validation."""
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr
    from monodetr_b200 import dataset as ds
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    from monodetr_b200.tester import Tester
    from monodetr_b200.trainer import Trainer
    world, rank = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl")
    os.chdir(a.out)                                 # Tester / Trainer write under "./" + save_path
    train_cfg = {"max_epoch": 1, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": f"w{world}_r{rank}"}
    torch.manual_seed(0)
    train_loader, test_loader = ds.build_dataloader(dict(DATASET, root_dir=a.root, batch_size=a.batch), workers=4)
    model, _ = build_monodetr(DEFAULT_MODEL_CFG)
    model = model.cuda()
    tester = Tester({"topk": 50, "threshold": 0.2}, model, test_loader, _Quiet(), train_cfg)
    passes = []
    for i in range(a.repeats + 1):
        _sync_barrier(world)
        t0 = time.perf_counter()
        tester.inference()
        ap = tester.evaluate()
        _sync_barrier(world)
        if i:
            passes.append(round(time.perf_counter() - t0, 3))
    # one Trainer epoch (training batches of --train-batch) with the tester attached
    train_loader.loader = torch.utils.data.DataLoader(train_loader.loader.dataset, batch_size=a.train_batch, shuffle=True,
                                                      num_workers=4, worker_init_fn=ds.my_worker_init_fn, drop_last=False,
                                                      collate_fn=ds._keep_lists)
    crit = build_criterion(CRIT_CFG).cuda().train()
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler({"warmup": True, "decay_rate": 0.1, "decay_list": [125, 165]}, opt, last_epoch=-1)
    trainer = Trainer(dict(train_cfg, max_epoch=2), model, opt, train_loader, test_loader, sched, warm, _Quiet(), crit, "bench")
    trainer.tester = tester
    epochs = []
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        for e in range(2):                          # the first epoch captures the graphs
            _sync_barrier(world)
            t0 = time.perf_counter()
            trainer.cfg["max_epoch"] = trainer.epoch + 1
            trainer.train()
            _sync_barrier(world)
            epochs.append(round(time.perf_counter() - t0, 3))
    if rank == 0:
        with open(os.path.join(a.out, f"w{world}.json"), "w") as f:
            json.dump({"validation_pass_s": passes, "car_ap3d_r40": ap, "trainer_epoch_with_validation_s": epochs[1:],
                       "first_epoch_with_capture_s": epochs[0], "val_batches_per_rank": -(-len(test_loader) // world),
                       "train_batches": len(train_loader)}, f)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def replicate_val(root, n):
    """Make the val split `n` images long by hard-linking the written ones (image, label, calib) under new ids: PNG
    encoding would dominate the run, and the timing does not depend on what the images show."""
    with open(os.path.join(root, "ImageSets", "val.txt")) as f:
        src = [x.strip() for x in f if x.strip()]
    new = ["%06d" % (900000 + k) for k in range(n)]
    for k, i in enumerate(new):
        for sub, ext in (("image_2", "png"), ("label_2", "txt"), ("calib", "txt")):
            os.link(os.path.join(root, "training", sub, f"{src[k % len(src)]}.{ext}"), os.path.join(root, "training", sub, f"{i}.{ext}"))
    with open(os.path.join(root, "ImageSets", "val.txt"), "w") as f:
        f.write("".join(i + "\n" for i in new))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--val", type=int, default=3769)
    ap.add_argument("--train", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--train-batch", type=int, default=8)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--worlds", type=int, nargs="+", default=[1, 2, 8])
    ap.add_argument("--worker", nargs=2, metavar=("ROOT", "OUT"))
    a = ap.parse_args()
    if a.worker:
        a.root, a.out = a.worker
        worker(a)
        return
    if not torch.cuda.is_available():
        raise SystemExit("bench_dist_validation: a CUDA device is required (nothing is measured without one)")
    import synthetic_kitti as sk
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "gpus_visible": torch.cuda.device_count(), "val_images": a.val, "train_images": a.train,
           "val_batch": a.batch, "train_batch": a.train_batch, "resolution": "1280x384", "worlds": {}}
    with tempfile.TemporaryDirectory() as tmp:
        root, out = os.path.join(tmp, "kitti"), os.path.join(tmp, "out")
        os.makedirs(out)
        t0 = time.perf_counter()
        sk.write_tree(root, n_train=a.train, n_val=64, n_test=1, seed=1)
        replicate_val(root, a.val)
        res["tree_write_s"] = round(time.perf_counter() - t0, 1)
        for w in a.worlds:
            if w > torch.cuda.device_count():
                res["worlds"][str(w)] = "not measured"
                continue
            cmd = [sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={w}", os.path.abspath(__file__),
                   "--val", str(a.val), "--batch", str(a.batch), "--train-batch", str(a.train_batch), "--repeats", str(a.repeats),
                   "--worker", root, out]
            subprocess.run(cmd, check=True, env=dict(os.environ, PYTHONPATH=ROOT))
            with open(os.path.join(out, f"w{w}.json")) as f:
                res["worlds"][str(w)] = json.load(f)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
