"""Drop-in for the reference's lib/helpers/tester_helper.py `Tester` in the validation pass of `Trainer.train`
(trainer_helper.py:97-100): `inference()` then `evaluate()`.

The reference decodes each batch on the host, writes one result file per image (`save_results`) and evaluates by reading
those files and the split's label files back (`KITTI_Dataset.eval`).  Here the decoded detections of every batch stay in a
device table (`kitti_eval.DeviceEvaluator`), the labels are parsed once per `Tester`, and `evaluate()` computes the AP from the
table with one host synchronisation.  The result files are still written under `<save_path>/<model_name>/outputs/data`, byte
for byte as the reference writes them, from one device->host copy.

Loader contract (the reference's): batches `(inputs, calibs, targets, info)` with `info['img_id']` and `info['img_size']`;
`dataset.idx_list / label_dir / writelist / class_name / cls_mean_size`.  The batch's `calibs` (P2 of each image, as the
val / test splits return them unchanged) feed the decode, instead of re-reading the calib files.
`save_results(results)` is kept for callers that decode on their own; `test()` (checkpoint loading) is not provided.
"""
import os

import torch

from . import kitti_eval


class Tester:
    def __init__(self, cfg, model, dataloader, logger, train_cfg=None, model_name="monodetr"):
        self.cfg = cfg
        self.model = model
        self.dataloader = dataloader
        dataset = dataloader.dataset
        self.class_name = dataset.class_name
        self.output_dir = os.path.join("./" + train_cfg["save_path"], model_name)
        self.dataset_type = cfg.get("type", "KITTI")
        if self.dataset_type != "KITTI":
            raise NotImplementedError("Tester: only the KITTI dataset type is implemented")
        self.device = kitti_eval._device()
        self.logger = logger
        self.train_cfg = train_cfg
        self.model_name = model_name
        ids = [int(i) for i in dataset.idx_list]
        self._slot = {img_id: s for s, img_id in enumerate(ids)}
        gt = None
        if getattr(dataset, "split", None) != "test":
            gt = kitti_eval.GroundTruth(kitti_eval.get_label_annos(dataset.label_dir, ids), ids, self.device)
        self.evaluator = kitti_eval.DeviceEvaluator(gt, dataset.writelist, topk=cfg["topk"], threshold=cfg.get("threshold", 0.2),
                                                    cls_mean_size=dataset.cls_mean_size, class_names=self.class_name,
                                                    image_ids=ids, device=self.device)

    def inference(self):
        torch.set_grad_enabled(False)
        self.model.eval()
        self.evaluator.reset()
        for inputs, calibs, targets, info in self.dataloader:
            inputs = inputs.to(self.device)
            calibs = calibs.to(self.device)
            img_sizes = info["img_size"].to(self.device)
            outputs = self.model(inputs, calibs, targets, img_sizes, dn_args=0)
            slots = [self._slot[int(i)] for i in info["img_id"]]
            self.evaluator.add(outputs, slots, img_sizes, calibs)
        self.logger.info("==> Saving ...")
        self.evaluator.write_results(os.path.join(self.output_dir, "outputs", "data"), self.class_name)

    def save_results(self, results):
        """The reference's save_results: {img_id: [[cls_id, alpha, x0, y0, x1, y1, h, w, l, X, Y, Z, ry, score], ...]} (what
        decode.decode_detections returns) -> <output_dir>/outputs/data/%06d.txt, one file per image, in the reference's format.
        `inference()` does not need it: it writes the same files from the device table."""
        output_dir = os.path.join(self.output_dir, "outputs", "data")
        os.makedirs(output_dir, exist_ok=True)
        for img_id, rows in results.items():
            with open(os.path.join(output_dir, "{:06d}.txt".format(img_id)), "w") as f:
                f.write(kitti_eval.result_file_text(rows, self.class_name))

    def evaluate(self):
        """Car AP3d R40 at moderate difficulty (0 when 'Car' is not in the writelist), with KITTI_Dataset.eval's log lines."""
        return self.evaluator.result(self.logger)
