"""GPU, two or more H100s, NCCL: `Tester.inference()` / `evaluate()` of the small golden model under torchrun with 2 ranks
against the same run with 1 rank, both in reproducible mode.  The result files must be byte-identical and the AP equal on
every rank.  Skips with fewer than two GPUs.

Run as a script (by torchrun), the file is the worker: `<file> <out_dir> <label_dir>`."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
N_IMG, BATCH = 14, 3                    # 5 batches, the last one short: rank 0 runs 3 and rank 1 runs 2
IDS = [3, 8, 15, 16, 42, 77, 80, 81, 99, 120, 121, 205, 300, 301]
NAMES = ["Pedestrian", "Car", "Cyclist"]


def _model_and_batches():
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from oracle import monodetr_torch as om
    g = np.load(os.path.join(HERE, "golden", "model_eval_small.npz"))
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG))
    model.load_state_dict(om.with_aliases(om.deterministic_state_dict()))
    images, calibs, sizes = om.synthetic_inputs(N_IMG, int(g["seed"]) + 1, H=int(g["H"]), W=int(g["W"]))
    batches = [(images[b:b + BATCH], calibs[b:b + BATCH], {}, {"img_id": torch.tensor(IDS[b:b + BATCH]), "img_size": sizes[b:b + BATCH]})
               for b in range(0, N_IMG, BATCH)]
    return model.cuda().eval(), batches


class _Loader:
    def __init__(self, dataset, batches):
        self.dataset, self.batches = dataset, batches

    def __iter__(self):
        return iter(self.batches)

    def __len__(self):
        return len(self.batches)


class _Log:
    def __init__(self):
        self.lines = []

    def info(self, s):
        self.lines.append(s)


def _worker(out_dir, label_dir):
    import types
    import torch.distributed as dist
    import monodetr_b200
    from monodetr_b200 import tester
    world = int(os.environ["WORLD_SIZE"])
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    if world > 1:
        dist.init_process_group("nccl")
    monodetr_b200.set_deterministic(True)
    model, batches = _model_and_batches()
    ds = types.SimpleNamespace(idx_list=["%06d" % i for i in IDS], label_dir=label_dir, writelist=["Car", "Pedestrian", "Cyclist"],
                               class_name=NAMES, cls_mean_size=np.zeros((3, 3), np.float32), split="val", max_objs=50)
    os.makedirs(os.path.join(out_dir, str(rank)), exist_ok=True)
    os.chdir(os.path.join(out_dir, str(rank)))
    log = _Log()
    t = tester.Tester({"topk": 50, "threshold": 0.0}, model, _Loader(ds, batches), log, {"save_path": "out"})
    t.inference()
    car = t.evaluate()
    with open("result.json", "w") as f:
        json.dump({"car": car, "log": log.lines}, f)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def _torchrun(world, out_dir, label_dir):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, HERE]))
    subprocess.run([sys.executable, "-m", "torch.distributed.run", "--standalone", f"--nproc_per_node={world}", __file__,
                    out_dir, label_dir], check=True, env=env, timeout=900)
    res = []
    for r in range(world):
        with open(os.path.join(out_dir, str(r), "result.json")) as f:
            res.append(json.load(f))
        data = os.path.join(out_dir, str(r), "out", "monodetr", "outputs", "data")
        res[-1]["files"] = {n: open(os.path.join(data, n), "rb").read() for n in sorted(os.listdir(data))} if os.path.isdir(data) else {}
    return res


@pytest.mark.gpu
def test_two_ranks_equal_one_rank(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from monodetr_b200 import kitti_eval as ke
    from test_validation_gpu import labels_near, write_file_path
    import monodetr_b200
    monodetr_b200.set_deterministic(True)
    try:
        model, batches = _model_and_batches()
        with torch.no_grad():                                          # labels near the model's own detections
            outs = [model(x.cuda(), c.cuda(), None, s["img_size"].cuda()) for x, c, _, s in batches]
        write_file_path(str(tmp_path / "ref"), [(o, s["img_size"].cuda(), c.cuda()) for o, (_, c, _, s) in zip(outs, batches)],
                        [IDS[b:b + BATCH] for b in range(0, N_IMG, BATCH)], np.zeros((3, 3), np.float32), thr=0.0)
    finally:
        monodetr_b200.set_deterministic(False)
    os.makedirs(tmp_path / "label_2")
    for i, text in zip(IDS, labels_near(ke.get_label_annos(str(tmp_path / "ref")), np.random.default_rng(2))):
        (tmp_path / "label_2" / ("%06d.txt" % i)).write_text(text)
    one = _torchrun(1, str(tmp_path / "w1"), str(tmp_path / "label_2"))[0]
    two = _torchrun(2, str(tmp_path / "w2"), str(tmp_path / "label_2"))
    assert one["car"] > 0 and len(one["files"]) == N_IMG
    assert two[0]["car"] == one["car"] and two[1]["car"] == one["car"]
    assert two[0]["log"] == one["log"] and two[0]["files"] == one["files"]
    assert two[1]["log"] == [] and two[1]["files"] == {}


if __name__ == "__main__":
    sys.path[:0] = [ROOT, HERE]
    _worker(sys.argv[1], sys.argv[2])
