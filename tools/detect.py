"""3D boxes for a folder of camera frames, written as the reference's Tester writes its result files.

    python tools/detect.py --config CFG --checkpoint CKPT --images DIR_OR_LIST --calib DIR_OR_FILE --out DIR [--batch N]

  --config      the reference's YAML config: `model` builds the network, `tester` gives topk / threshold and `dataset`
                meanshape (monodetr_b200.detect.Detector.from_config)
  --checkpoint  a checkpoint in the reference's format (its `model_state` is loaded)
  --images      a directory (every .png / .jpg / .jpeg in it, in name order) or a text file listing one image path per line
                (relative paths are taken from the list's directory); 8-bit RGB images, decoded with Pillow
  --calib       a directory holding <image stem>.txt per image, or one KITTI calib file for every image; P2 is its third line
  --out         <out>/<name>.txt per image: %06d.txt for a numeric stem (KITTI ids), <stem>.txt otherwise
  --batch       frames per forward (default: the config's dataset batch_size, else 16)

The lines are `kitti_eval.result_file_text` of the decoded rows with the class names of the KITTI dataset (Pedestrian, Car,
Cyclist), so for the same model, frames and batches the bytes are those Tester.inference() writes under outputs/data.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

IMAGE_EXTS = (".png", ".jpg", ".jpeg")


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description="Detect 3D boxes on camera frames with a MonoDETR checkpoint")
    ap.add_argument("--config", required=True)
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--images", required=True, help="a directory of images, or a text file listing image paths")
    ap.add_argument("--calib", required=True, help="a directory of <stem>.txt calib files, or one calib file for every image")
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=None)
    args = ap.parse_args(argv)
    if args.batch is not None and args.batch < 1:
        ap.error("--batch must be at least 1")
    return args


def image_paths(spec):
    """The images of --images, in order."""
    if os.path.isdir(spec):
        paths = [os.path.join(spec, f) for f in sorted(os.listdir(spec)) if f.lower().endswith(IMAGE_EXTS)]
    else:
        base = os.path.dirname(os.path.abspath(spec))
        with open(spec) as f:
            paths = [os.path.join(base, ln.strip()) for ln in f if ln.strip()]
    if not paths:
        raise ValueError(f"--images {spec}: no images")
    return paths


def stem(path):
    return os.path.splitext(os.path.basename(path))[0]


def result_name(path):
    """%06d.txt for a numeric stem (as the Tester names KITTI ids), <stem>.txt otherwise."""
    s = stem(path)
    return "%06d.txt" % int(s) if s.isdigit() else s + ".txt"


def calib_paths(paths, spec):
    """The calib file of each image: <spec>/<stem>.txt when --calib is a directory, else --calib itself."""
    if os.path.isdir(spec):
        return [os.path.join(spec, stem(p) + ".txt") for p in paths]
    return [spec] * len(paths)


def main(argv=None):
    import numpy as np
    import yaml

    from monodetr_b200 import kitti_eval
    from monodetr_b200.dataset import decode_image, read_image_sizes
    from monodetr_b200.detect import Detector
    from monodetr_b200.labels import CLASS_NAMES, parse_calib_file

    args = parse_args(argv)
    with open(args.config) as f:
        cfg = yaml.load(f, Loader=yaml.Loader)
    paths = image_paths(args.images)
    names = [result_name(p) for p in paths]
    if len(set(names)) != len(names):
        raise ValueError("--images: two images map to the same result file name")
    P2 = np.stack([parse_calib_file(p) for p in calib_paths(paths, args.calib)])
    sizes = read_image_sizes(paths)                         # every header is checked before the first decode
    batch = args.batch or int((cfg.get("dataset") or {}).get("batch_size", 16))
    det = Detector.from_config(cfg, args.checkpoint, max_batch=batch, max_frame=tuple(int(v) for v in sizes.max(0)))
    os.makedirs(args.out, exist_ok=True)
    for b0 in range(0, len(paths), batch):
        frames = [decode_image(p) for p in paths[b0:b0 + batch]]
        for name, rows in zip(names[b0:b0 + batch], det.detect(frames, P2[b0:b0 + batch])):
            with open(os.path.join(args.out, name), "w") as f:
                f.write(kitti_eval.result_file_text(rows.tolist(), CLASS_NAMES))
    print(f"{len(paths)} images -> {args.out}")


if __name__ == "__main__":
    main()
