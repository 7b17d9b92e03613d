"""Time the KITTI validation pass after the forward: the result-file path against the device path, on a val-sized set.

    python tools/bench_validation.py [--images 3769] [--batch 32] [--repeats 3] [--model]

Decode inputs are seeded synthetic head outputs (oracle.decode.synthetic_heads), labels are KITTI-like and lie near the
detections.  Both paths evaluate Car, Pedestrian and Cyclist:
  file    per batch decode_detections (one device->host copy each), the reference's save_results formatting into one file per
          image, then kitti_eval.evaluate (parse the result and label files, pack, upload, eval);
  device  per batch DeviceEvaluator.add (extract + decode + collect, no synchronisation), then result() (one copy of the
          per-image counts, compaction, eval) on labels parsed once (GroundTruth);
  tester  what monodetr_b200.tester.Tester runs per pass: the device path plus write_results (one copy of the table, the
          result files formatted and written).
--model puts the eval forward of the default model (random weights, 384x1280) in front of both, for the whole pass.
After one warm-up of each, the two paths alternate `--repeats` times; each is timed with host clocks around work that ends in
a device synchronisation.  Prints one JSON line with the GPU name and power limit read in the same run."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from monodetr_b200 import decode  # noqa: E402
from monodetr_b200 import kitti_eval as ke  # noqa: E402
from oracle import decode as od  # noqa: E402

NAMES = ["Pedestrian", "Car", "Cyclist"]
CLASSES = ["Car", "Pedestrian", "Cyclist"]


def batches(n_img, B, dev):
    out = []
    for k, b0 in enumerate(range(0, n_img, B)):
        h = od.synthetic_heads(1000 + k, min(B, n_img - b0), 50)
        heads = {"pred_logits": h["logits"], "pred_boxes": h["boxes"], "pred_3d_dim": h["dim3"], "pred_depth": h["depth"],
                 "pred_angle": h["angle"]}
        out.append(({k2: torch.from_numpy(v).to(dev) for k2, v in heads.items()}, torch.from_numpy(h["img_size"]).to(dev),
                    torch.from_numpy(h["P2"]).to(dev)))
    return out


def write_labels(label_dir, res_dir, ids, rng):
    os.makedirs(label_dir, exist_ok=True)
    for i, a in zip(ids, ke.get_label_annos(res_dir)):
        lines = []
        for j in range(len(a["name"])):
            if rng.random() < 0.5:
                continue
            l, h, w = a["dimensions"][j]
            lines.append("{} 0.00 0 {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f}\n".format(
                a["name"][j], a["alpha"][j], *(a["bbox"][j] + rng.normal(0, 2, 4)), h, w, l, *(a["location"][j] + rng.normal(0, 0.1, 3)),
                a["rotation_y"][j]))
        with open(os.path.join(label_dir, "%06d.txt" % i), "w") as f:
            f.write("".join(lines))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_validation: needs a CUDA device")
    dev = torch.device("cuda", 0)
    ids = list(range(a.images))
    data = batches(a.images, a.batch, dev)
    bids = [ids[b0:b0 + a.batch] for b0 in range(0, a.images, a.batch)]
    mean = od.synthetic_heads(0, 1, 1)["mean_size"]
    model = None
    if a.model:
        from monodetr_b200 import build_monodetr
        from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
        torch.manual_seed(0)
        model = build_monodetr(dict(DEFAULT_MODEL_CFG))[0].to(dev).eval()
        images = torch.randn(a.batch, 3, 384, 1280, device=dev)

    def heads_of(k):
        out, size, P2 = data[k]
        if model is None:
            return out
        with torch.no_grad():
            full = model(images[:len(bids[k])], P2, None, size)
        return {key: full[key] for key in out}

    tmp = tempfile.mkdtemp(prefix="bench_validation_")

    class Quiet:
        def info(self, s):
            pass

    label_dir = os.path.join(tmp, "label_2")

    def file_path(run):
        res_dir = os.path.join(tmp, f"res{run}")
        os.makedirs(res_dir)
        for k, (out, size, P2) in enumerate(data):
            dets = decode.extract_dets_from_outputs(heads_of(k), topk=50)
            res = decode.decode_detections(dets, {"img_id": bids[k], "img_size": size}, P2, mean, 0.2)
            for img_id, rows in res.items():                   # tester_helper.py:118-132
                with open(os.path.join(res_dir, "{:06d}.txt".format(img_id)), "w") as f:
                    for r in rows:
                        f.write("{} 0.0 0".format(NAMES[int(r[0])]))
                        for v in r[1:]:
                            f.write(" {:.2f}".format(v))
                        f.write("\n")
        if not os.path.exists(label_dir):
            write_labels(label_dir, res_dir, ids, np.random.default_rng(1))
        return ke.evaluate(res_dir, label_dir, ids, CLASSES, Quiet())

    run_ctr = [0]

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v = fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, v

    def file_once():
        run_ctr[0] += 1
        return file_path(run_ctr[0])

    file_once()                                                     # warm-up; also writes the labels
    gt = ke.GroundTruth(ke.get_label_annos(label_dir, ids), ids)
    ev = ke.DeviceEvaluator(gt, CLASSES, cls_mean_size=mean)

    def device_once():
        ev.reset()
        for k, (out, size, P2) in enumerate(data):
            ev.add(heads_of(k), list(range(k * a.batch, k * a.batch + len(bids[k]))), size, P2)
        return ev.result(Quiet())

    def tester_once():
        run_ctr[0] += 1
        v = device_once()
        ev.write_results(os.path.join(tmp, f"tester{run_ctr[0]}"), NAMES)
        return v

    device_once()
    tester_once()
    file_s, dev_s, tester_s, vals = [], [], [], set()
    for _ in range(a.repeats):
        for fn, acc in ((file_once, file_s), (device_once, dev_s), (tester_once, tester_s)):
            t, v = timed(fn)
            acc.append(round(t, 3))
            vals.add(v)
    out = {"images": a.images, "batch": a.batch, "model_forward_included": a.model, "file_path_s": file_s,
           "device_path_s": dev_s, "tester_path_s": tester_s,
           "speedup_median": round(float(np.median(file_s) / np.median(dev_s)), 1),
           "tester_speedup_median": round(float(np.median(file_s) / np.median(tester_s)), 1),
           "same_car_ap3d_r40": len(vals) == 1, "car_ap3d_r40": float(next(iter(vals))), "gpu": torch.cuda.get_device_name(0)}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
