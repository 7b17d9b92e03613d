"""Training criterion on the device (SURVEY.md 8 f1) behind the reference's classes.

  HungarianMatcher(cost_class, cost_3dcenter, cost_bbox, cost_giou)            lib/models/monodetr/matcher.py:14-104
  SetCriterion(num_classes, matcher, weight_dict, focal_alpha, losses, group_num).forward(outputs, targets)
                                                                                lib/models/monodetr/monodetr.py:297-532
  build_matcher(cfg) / build_criterion(cfg)                                     matcher.py:107-112, monodetr.py:575-612

Same constructor arguments, same `weight_dict`, same keys and values in the returned dict (`loss_ce`, `class_error`, `loss_bbox`,
`loss_giou`, `cardinality_error`, `loss_depth`, `loss_dim`, `loss_angle`, `loss_center`, `loss_depth_map` and the `_0`, `_1`
aux copies), same gradients -- but the whole thing is five kernel launches forward and two backward (csrc/criterion.cu) with no
host synchronisation: the assignment problems are solved on the GPU (one warp each) instead of `C.cpu()` + scipy, `num_boxes`
stays a device scalar, and `targets` may be the data loader's PADDED batch dict (with `mask_2d`) so that
`Trainer.prepare_targets`' boolean-index compaction (trainer_helper.py:175-186, one sync per image and key) is not needed.
The reference's list-of-dicts form is accepted too.  There is no CPU path.
"""
import torch
import torch.distributed as dist
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib

NUM_LOSSES = 10                 # MDB_CRITERION_NUM_LOSSES
MAX_LAYERS = 6                  # MDB_CRITERION_MAX_LAYERS: decoder layers (final outputs + auxiliary outputs) per call
MAX_QUERIES = 300               # queries per group the match kernel takes (csrc/criterion.cu)
BASE_QUERIES = 64               # queries per group a SetCriterion takes unless it is built for more (max_queries)
(CE, CLASS_ERROR, BBOX, GIOU, CARDINALITY, DEPTH, DIM, ANGLE, CENTER, DEPTH_MAP) = range(NUM_LOSSES)
_NAMES = {CE: "loss_ce", CLASS_ERROR: "class_error", BBOX: "loss_bbox", GIOU: "loss_giou", CARDINALITY: "cardinality_error",
          DEPTH: "loss_depth", DIM: "loss_dim", ANGLE: "loss_angle", CENTER: "loss_center", DEPTH_MAP: "loss_depth_map"}
_GROUPS = {"labels": (CE, CLASS_ERROR), "boxes": (BBOX, GIOU), "cardinality": (CARDINALITY,), "depths": (DEPTH,), "dims": (DIM,),
           "angles": (ANGLE,), "center": (CENTER,), "depth_map": (DEPTH_MAP,)}
_PRED_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle")
_TGT_KEYS = ("labels", "boxes", "boxes_3d", "depth", "size_3d", "heading_bin", "heading_res")


class HungarianMatcher(nn.Module):
    """Holds the four cost weights (matcher.py:21-33); the assignment itself runs inside SetCriterion's match kernel."""

    def __init__(self, cost_class: float = 1, cost_3dcenter: float = 1, cost_bbox: float = 1, cost_giou: float = 1):
        super().__init__()
        self.cost_class, self.cost_3dcenter, self.cost_bbox, self.cost_giou = cost_class, cost_3dcenter, cost_bbox, cost_giou
        assert cost_class != 0 or cost_bbox != 0 or cost_giou != 0, "all costs cant be 0"

    @torch.no_grad()
    def forward(self, outputs, targets, group_num=11):
        """Reference signature and result: list (per image) of (query indices, target indices) int64 tensors -- on the device."""
        tgt = pack_targets(targets, outputs["pred_logits"].device)
        st = _prepare(tgt)
        match, _ = _match(self, [outputs], tgt, st, group_num)
        B, Gmax = tgt["mask"].shape
        m = match[0]                                                       # (B, group, Gmax)
        res = []
        for b in range(B):                                                 # (this convenience path synchronises; the criterion does not)
            sel = m[b] >= 0
            j = torch.arange(Gmax, device=m.device).expand_as(m[b])[sel]
            res.append((m[b][sel].long(), j))
        return res


def build_matcher(cfg):
    return HungarianMatcher(cost_class=cfg["set_cost_class"], cost_bbox=cfg["set_cost_bbox"], cost_3dcenter=cfg["set_cost_3dcenter"],
                            cost_giou=cfg["set_cost_giou"])


def pack_targets(targets, device, max_objs=None):
    """Loader batch dict (padded (B, Gmax, ...) arrays + `mask_2d`) or the reference's list of per-image dicts -> dense device
    tensors in the dtypes the kernels read.  Only host-known shapes are used: no synchronisation."""
    if isinstance(targets, dict) and "mask" in targets and targets.get("_packed"):
        return targets
    if isinstance(targets, (list, tuple)):
        B = len(targets)
        G = max_objs or max([int(t["labels"].shape[0]) for t in targets] + [1])
        dense = {k: None for k in _TGT_KEYS}
        mask = torch.zeros(B, G, dtype=torch.uint8, device=device)
        for k in _TGT_KEYS:
            tail = tuple(targets[0][k].shape[1:])
            dense[k] = torch.zeros((B, G) + tail, dtype=torch.float32, device=device)
        for b, t in enumerate(targets):
            n = int(t["labels"].shape[0])
            if n:
                mask[b, :n] = 1
                for k in _TGT_KEYS:
                    dense[k][b, :n] = t[k].to(device=device, dtype=torch.float32)
        src = dense
    else:
        src = targets
        mask = targets["mask_2d"].to(device=device, dtype=torch.uint8)
    B, G = mask.shape
    if G > 64:
        raise ValueError("criterion: at most 64 objects per image")
    f = lambda k, *shape: src[k].to(device=device, dtype=torch.float32).reshape(B, G, *shape).contiguous()  # noqa: E731
    i = lambda k: src[k].to(device=device).reshape(B, G).to(torch.int32).contiguous()  # noqa: E731
    return {"_packed": True, "mask": mask.contiguous(), "labels": i("labels"), "boxes2d": f("boxes", 4), "boxes3d": f("boxes_3d", 6),
            "depth": f("depth"), "size3d": f("size_3d", 3), "hbin": i("heading_bin"), "hres": f("heading_res")}


def _prepare(tgt):
    B, G = tgt["mask"].shape
    dev = tgt["mask"].device
    st = {"tlist": torch.empty(B, G, dtype=torch.int32, device=dev), "count": torch.empty(B, dtype=torch.int32, device=dev),
          "total": torch.empty(1, dtype=torch.float32, device=dev), "world": 1.0}
    _lib.call("mdb_criterion_prepare", tgt["mask"], B, G, st["tlist"], st["count"], st["total"])
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(st["total"])                                       # monodetr.py:506-508
        st["world"] = float(dist.get_world_size())
    return st


def _layer_tensors(layers):
    return [[l[k].detach().float().contiguous() for l in layers] for k in _PRED_KEYS]


def _match(matcher, layers, tgt, st, group):
    logits, boxes = ([l[k].detach().float().contiguous() for l in layers] for k in ("pred_logits", "pred_boxes"))
    B, Q, C = logits[0].shape
    G = tgt["mask"].shape[1]
    L = len(layers)
    if Q % group:
        raise ValueError("criterion: the number of queries must be a multiple of group_num")
    dev = logits[0].device
    match = torch.empty(L, B, group, G, dtype=torch.int32, device=dev)
    tclass = torch.empty(L, B, Q, dtype=torch.int32, device=dev)
    _lib.call("mdb_criterion_match_f32", L, logits, boxes, tgt["labels"], tgt["boxes3d"], st["tlist"], st["count"], B, Q, C, group, G,
              float(matcher.cost_class), float(matcher.cost_3dcenter), float(matcher.cost_bbox), float(matcher.cost_giou), match, tclass)
    return match, tclass


def _depth_layout(x):
    """(B, D, H, W) logits -> (tensor to address, stride_b, stride_pix, stride_c): NHWC storage (the model's) or NCHW."""
    B, D, H, W = x.shape
    if x.permute(0, 2, 3, 1).is_contiguous():
        return x, H * W * D, D, 1
    x = x.contiguous()
    return x, D * H * W, 1, H * W


class _CriterionFn(Function):
    """(depth-map logits or None, 5 prediction tensors per decoder layer) -> losses (L, 10)."""

    @staticmethod
    def forward(ctx, crit, tgt, group, depth_logits, *preds):
        L = len(preds) // 5
        layers = [dict(zip(_PRED_KEYS, preds[5 * l:5 * l + 5])) for l in range(L)]
        per_key = _layer_tensors(layers)
        logits = per_key[0]
        B, Q, C = logits[0].shape
        G = tgt["mask"].shape[1]
        dev = logits[0].device
        with torch.cuda.device(dev):
            st = _prepare(tgt)
            match, tclass = _match(crit.matcher, layers, tgt, st, group)
            pix_loss, npix, dl = None, 0, None
            if depth_logits is not None:
                x, sb, sp, sc = _depth_layout(depth_logits.detach().float())
                _, D, H, W = x.shape
                npix = B * H * W
                pix_loss = torch.empty(npix, dtype=torch.float32, device=dev)
                sx, sy = crit.depth_map_scale
                dl = (x, sb, sp, sc, D, H, W, float(sx), float(sy))
                _lib.call("mdb_criterion_depth_map_f32", x, sb, sp, sc, tgt["boxes2d"], tgt["depth"], st["tlist"], st["count"], B, H, W,
                          D - 1, G, float(sx), float(sy), crit.depth_min, crit.depth_max, crit.ddn_alpha, crit.fg_weight, crit.bg_weight,
                          pix_loss, None, None)
            losses = torch.empty(L, NUM_LOSSES, dtype=torch.float32, device=dev)
            aux = torch.empty(L, dtype=torch.float32, device=dev)
            # launches=2 for one kernel keeps the forward's count at 4 + depth, the figure step launch totals are compared against
            _lib.call("mdb_criterion_losses_f32", L, *per_key, tgt["labels"], tgt["boxes3d"], tgt["depth"], tgt["size3d"], tgt["hbin"],
                      tgt["hres"], st["tlist"], st["count"], st["total"], match, tclass, pix_loss, npix, B, Q, C, group, G,
                      float(crit.focal_alpha), st["world"], losses, aux, launches=2)
        ctx.state = (crit, tgt, st, match, tclass, per_key, dl, group, aux, (B, Q, C, G, L))
        ctx.mark_non_differentiable(match)
        return losses, match

    @staticmethod
    @once_differentiable
    def backward(ctx, glosses, _gmatch):
        crit, tgt, st, match, tclass, per_key, dl, group, aux, (B, Q, C, G, L) = ctx.state
        glosses = glosses.contiguous().float()
        grads = [[torch.empty_like(t) for t in per_key[k]] for k in range(5)]
        dev = glosses.device
        with torch.cuda.device(dev):
            _lib.call("mdb_criterion_losses_backward_f32", L, *per_key, tgt["labels"], tgt["boxes3d"], tgt["depth"], tgt["size3d"],
                      tgt["hbin"], tgt["hres"], st["tlist"], st["count"], st["total"], match, tclass, B, Q, C, group, G,
                      float(crit.focal_alpha), st["world"], glosses, aux, *grads)
            gdepth = None
            if dl is not None:
                x, sb, sp, sc, D, H, W, sx, sy = dl
                gdepth = torch.empty_like(x)
                gw = glosses[0, DEPTH_MAP:DEPTH_MAP + 1]
                _lib.call("mdb_criterion_depth_map_f32", x, sb, sp, sc, tgt["boxes2d"], tgt["depth"], st["tlist"], st["count"], B, H, W,
                          D - 1, G, sx, sy, crit.depth_min, crit.depth_max, crit.ddn_alpha, crit.fg_weight, crit.bg_weight, None, gw, gdepth)
        flat = []
        for l in range(L):
            flat += [grads[k][l] for k in range(5)]
        return (None, None, None, gdepth) + tuple(flat)


class SetCriterion(nn.Module):
    """monodetr.py:297-532.  `targets`: the loader's padded batch dict (keys labels, boxes, boxes_3d, depth, size_3d, heading_bin,
    heading_res, mask_2d) or the list of per-image dicts `Trainer.prepare_targets` builds."""

    def __init__(self, num_classes, matcher, weight_dict, focal_alpha, losses, group_num=11, depth_map_scale=(80, 24),
                 max_queries=BASE_QUERIES):
        super().__init__()
        if not BASE_QUERIES <= max_queries <= MAX_QUERIES:
            raise NotImplementedError(f"SetCriterion: max_queries={max_queries}: the matcher takes {BASE_QUERIES} to {MAX_QUERIES}")
        self.num_classes = num_classes
        # Queries per group this criterion accepts.  64 unless the model it is built for has more (build_criterion sets it from
        # cfg["num_queries"]), so that a criterion built from the loss settings alone keeps its 64-query limit.
        self.max_queries = max_queries
        self.matcher = matcher
        self.weight_dict = weight_dict
        self.losses = losses
        self.focal_alpha = focal_alpha
        self.group_num = group_num
        self.depth_map_scale = depth_map_scale          # monodetr.py:462 hard-codes the 1280x384 / 16 map: (80, 24)
        self.ddn_alpha, self.fg_weight, self.bg_weight = 0.25, 13.0, 1.0            # ddn_loss.py:14-19
        self.depth_min, self.depth_max = 1e-3, 60.0                                  # ddn_loss.py:68
        for l in losses:
            if l not in _GROUPS:
                raise AssertionError(f"do you really want to compute {l} loss?")
        self.last_indices = None

    def forward(self, outputs, targets, mask_dict=None):
        logits = outputs["pred_logits"]
        if not logits.is_cuda:
            raise RuntimeError("SetCriterion: CUDA tensors required (not implemented on the CPU)")
        if logits.shape[-1] != self.num_classes:
            raise ValueError("SetCriterion: pred_logits has a different number of classes")
        tgt = pack_targets(targets, logits.device)
        group = self.group_num if self.training else 1
        layers = [outputs] + list(outputs.get("aux_outputs", []))
        if len(layers) > MAX_LAYERS:
            raise ValueError(f"SetCriterion: at most {MAX_LAYERS - 1} auxiliary outputs")
        Q = logits.shape[1]
        if Q % group == 0 and Q // group > self.max_queries:
            raise RuntimeError(f"SetCriterion: {Q // group} queries per group, but this criterion takes at most {self.max_queries}; "
                               "build it with build_criterion(cfg) from a model section whose num_queries covers them")
        depth_logits = outputs["pred_depth_map_logits"] if "depth_map" in self.losses else None
        preds = [l[k] for l in layers for k in _PRED_KEYS]
        losses, match = _CriterionFn.apply(self, tgt, group, depth_logits, *preds)
        self.last_indices = match                                            # (L, B, group, Gmax) matched query per valid target, -1 = none
        self._last_losses = losses
        want = [k for l in self.losses for k in _GROUPS[l]]
        out = {}
        for li in range(len(layers)):
            for k in want:
                if li > 0 and k in (DEPTH_MAP, CLASS_ERROR):
                    continue                                                 # monodetr.py:519-527
                out[_NAMES[k] + ("" if li == 0 else f"_{li - 1}")] = losses[li, k]
        return out

    def weighted_sum(self):
        return weighted_sum(self)


def _weight_matrix(crit, L, device):
    key = (L, str(device), tuple(sorted(crit.weight_dict.items())))
    if getattr(crit, "_wm_key", None) != key:
        w = torch.zeros(L, NUM_LOSSES)
        want = {k for l in crit.losses for k in _GROUPS[l]}
        for li in range(L):
            for k in want:
                if li > 0 and k in (DEPTH_MAP, CLASS_ERROR):
                    continue
                w[li, k] = float(crit.weight_dict.get(_NAMES[k] + ("" if li == 0 else f"_{li - 1}"), 0.0))
        crit._wm, crit._wm_key = w.to(device), key
    return crit._wm


def weighted_sum(crit):
    """sum(losses[k] * weight_dict[k]) of the criterion's LAST forward (what lib/helpers/trainer_helper.py:141-143 computes with a
    Python loop over the dict: ~26 multiplies + adds and as many autograd nodes) as one multiply + one reduction."""
    losses = crit._last_losses
    return (losses * _weight_matrix(crit, losses.shape[0], losses.device)).sum()


class LossLog:
    """The trainer's loss log (lib/helpers/trainer_helper.py:145-152) without a host synchronisation per step.  `push()` -- one
    launch, graph-safe -- appends the weighted loss table of the criterion's last forward to a device ring; `fetch(step)` starts
    an asynchronous copy of that step's record into pinned memory and returns a handle whose `ready()` polls an event behind
    the copy and whose `read()` gives the reference's log dict: every term of `weight_dict` as `(loss * weight).item()` would
    return it, in the criterion's dict order, and `loss_detr` = their sum accumulated in Python floats in that order."""

    def __init__(self, crit, n_layers, device, slots=64):
        self.crit, self.L, self.slots, self.n = crit, n_layers, slots, n_layers * NUM_LOSSES
        self.ring = torch.zeros(slots, self.n + 1, dtype=torch.float32, device=device)
        self.counter = torch.zeros(1, dtype=torch.int64, device=device)
        self.pushed = 0                                                       # host mirror of the device counter
        want = [k for l in crit.losses for k in _GROUPS[l]]
        self.terms = []                                                       # (name, index into the flattened table)
        for li in range(n_layers):
            for k in want:
                name = _NAMES[k] + ("" if li == 0 else f"_{li - 1}")
                if not (li > 0 and k in (DEPTH_MAP, CLASS_ERROR)) and name in crit.weight_dict:
                    self.terms.append((name, li * NUM_LOSSES + k))

    def push(self):
        losses = self.crit._last_losses
        _lib.call("mdb_trainlog_push_f32", losses, _weight_matrix(self.crit, self.L, losses.device), self.n, self.ring, self.slots,
                  self.counter)
        if not (torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()):
            self.pushed += 1                                                  # a captured push runs at replay: see replayed()

    def replayed(self):
        """Tell the host mirror that a graph holding a captured `push()` has been replayed once."""
        self.pushed += 1

    def fetch(self, step):
        """`step`: 0 for the first push ever, 1 for the second, ...; at most `slots` pushes may have followed it."""
        if not 0 <= self.pushed - 1 - step < self.slots:
            raise ValueError("LossLog.fetch: that step is no longer in the ring")
        rec = self.ring[step % self.slots]
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        if world > 1:                                                          # misc.reduce_dict: the mean over ranks
            rec = rec.clone()
            dist.all_reduce(rec)
            rec /= world
        host = torch.empty(self.n + 1, dtype=torch.float32, pin_memory=rec.device.type == "cuda")
        host.copy_(rec, non_blocking=True)
        event = torch.cuda.Event() if rec.device.type == "cuda" else None
        if event is not None:
            event.record()
        return _LogRecord(host, event, sorted(self.terms) if world > 1 else self.terms)


class _LogRecord:
    def __init__(self, host, event, terms):
        self.host, self.event, self.terms = host, event, terms

    def ready(self):
        return self.event is None or self.event.query()

    def read(self):
        if self.event is not None and not self.event.query():
            self.event.synchronize()
        values, log, total = self.host.tolist(), {}, 0
        for name, i in self.terms:
            log[name] = values[i]
            total += log[name]
        log["loss_detr"] = total
        return log


def build_weight_dict(cfg):
    """monodetr.py:578-601 (without the dn terms, which need use_dn -- SURVEY.md: not on the path)."""
    w = {"loss_ce": cfg["cls_loss_coef"], "loss_bbox": cfg["bbox_loss_coef"], "loss_giou": cfg["giou_loss_coef"],
         "loss_dim": cfg["dim_loss_coef"], "loss_angle": cfg["angle_loss_coef"], "loss_depth": cfg["depth_loss_coef"],
         "loss_center": cfg["3dcenter_loss_coef"], "loss_depth_map": cfg["depth_map_loss_coef"]}
    if cfg.get("aux_loss", True):
        aux = {}
        for i in range(cfg.get("dec_layers", 3) - 1):
            aux.update({k + f"_{i}": v for k, v in w.items()})
        aux.update({k + "_enc": v for k, v in w.items()})
        w.update(aux)
    return w


def build_criterion(cfg):
    losses = ["labels", "boxes", "cardinality", "depths", "dims", "angles", "center", "depth_map"]        # monodetr.py:603
    return SetCriterion(cfg["num_classes"], matcher=build_matcher(cfg), weight_dict=build_weight_dict(cfg), focal_alpha=cfg["focal_alpha"],
                        losses=losses, max_queries=max(BASE_QUERIES, cfg.get("num_queries", 50)))
