"""TEST INFRASTRUCTURE shared by tools/gen_golden_trainer.py and the trainer tests: a tiny model, criterion, loader, tester and
logger with the interfaces the reference's `Trainer` uses, small enough to run the whole training loop on the CPU in a second."""
import torch
from torch import nn

N_BATCHES = 32            # the log block is printed for batches 0 and 30
CFG = {"max_epoch": 7, "save_frequency": 1, "save_all": True, "use_dn": False, "save_path": "out"}
OPT_CFG = {"type": "adamw", "lr": 0.01, "weight_decay": 0.01}
SCHED_CFG = {"warmup": True, "decay_rate": 0.1, "decay_list": [5, 6]}
AP_SCRIPT = [0.1, 0.3, 0.2, 0.3, 0.5, 0.4, 0.45]


class StubModel(nn.Module):
    """Biases, weights and a layer that never receives a gradient (its name is one `FlatGradBucket` leaves out)."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(3)
        self.a = nn.Linear(4, 3)
        self.sa_v_proj = nn.Linear(2, 2)
        self.b = nn.Linear(3, 2)
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)

    def forward(self, images, calibs, targets, img_sizes, dn_args=None):
        return {"x": self.b(torch.tanh(self.a(images)))}


class StubCriterion(nn.Module):
    weight_dict = {"loss_ce": 2.0, "loss_bbox": 5.0, "loss_ce_0": 2.0, "loss_bbox_0": 5.0, "loss_unused": 1.0}

    def forward(self, outputs, targets, mask_dict=None):
        x = outputs["x"]
        n = sum(int(t["labels"].shape[0]) for t in targets)          # the list of per-image dicts `prepare_targets` builds
        return {"loss_ce": (x ** 2).mean() * 3, "class_error": x.detach().abs().max(), "loss_bbox": x.abs().mean() + 0.01 * n,
                "loss_ce_0": ((x - 1) ** 2).mean(), "loss_bbox_0": (x - 1).abs().mean()}


def make_loader(seed=0, n_batches=N_BATCHES, batch=2):
    """A list of `(inputs, calibs, targets, info)`; the last batch is short, as with `drop_last=False`."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n_batches):
        b = batch if i < n_batches - 1 else 1
        mask = torch.rand(b, 5, generator=g) < 0.5
        targets = {"labels": torch.randint(0, 3, (b, 5), generator=g), "mask_2d": mask, "img_size": torch.full((b, 2), 100.0),
                   "boxes": torch.rand(b, 5, 4, generator=g)}
        out.append((torch.randn(b, 4, generator=g) + 0.1 * rank_shift(), torch.eye(3, 4).expand(b, 3, 4).clone(), targets, {}))
    return out


def rank_shift():
    import torch.distributed as dist
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


class StubTester:
    def __init__(self, script=AP_SCRIPT):
        self.script, self.calls = list(script), 0

    def inference(self):
        self.calls += 1

    def evaluate(self):
        return self.script[self.calls - 1]


class ListLogger:
    def __init__(self):
        self.lines = []

    def info(self, msg):
        self.lines.append(str(msg))
