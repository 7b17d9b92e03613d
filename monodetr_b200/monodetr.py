"""MonoDETR top module -- mirror of lib/models/monodetr/monodetr.py (MonoDETR :28-293, MLP :535-547, build :550-614)
with identical constructor arguments, parameter names (state_dict keys incl. the decoder aliases :129-131),
initialisation rules and forward signature / output dict (:150, :270-283), running on the sm_90a kernels.

The configs/monodetr.yaml branch (with_box_refine=True, two_stage=False, two_stage_dino=False) is implemented with and without
the anchor-box queries (use_dab); use_dn changes nothing in the reference model.  two_stage / two_stage_dino / with_box_refine=False
raise NotImplementedError instead of silently differing.
"""
import copy
import math

import torch
import torch.nn.functional as F
from torch import nn

from . import functional as Fn, kernels as K, tc
from .backbone import build_backbone
from .depth_predictor import DepthPredictor
from .depthaware_transformer import MLP, build_depthaware_transformer, inverse_sigmoid


MAX_QUERIES = 300               # queries per group the device matcher takes (csrc/criterion.cu)


def head_stream(lvl):
    """Branch stream index of decoder level `lvl`'s prediction heads: 1-3 for levels 0-2, 25 and up for deeper levels (clear of
    the decoder's branches, depthaware_transformer.ahead_streams, and of the neck's 15-18)."""
    return 1 + lvl if lvl < 3 else 25 + (lvl - 3)


def _get_clones(module, N):
    return nn.ModuleList([copy.deepcopy(module) for _ in range(N)])


class _ProjGN(nn.Sequential):
    """input_proj entry: Sequential(Conv2d, GroupNorm(32, hidden)) (reference :83-91) with an NHWC forward."""

    def forward(self, x):
        conv, gn = self[0], self[1]
        y = Fn.conv2d_nhwc(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0])
        return Fn.groupnorm_nhwc(y, gn.weight, gn.bias, gn.num_groups, gn.eps, False)


class MonoDETR(nn.Module):
    """Monocular 3D detector; same constructor as the reference (:30-31)."""

    def __init__(self, backbone, depthaware_transformer, depth_predictor, num_classes, num_queries, num_feature_levels,
                 aux_loss=True, with_box_refine=False, two_stage=False, init_box=False, use_dab=False, group_num=11,
                 two_stage_dino=False):
        super().__init__()
        if two_stage or two_stage_dino:
            raise NotImplementedError("two_stage / two_stage_dino are not implemented: the reference itself fails with them "
                                      "(two_stage in the training forward, two_stage_dino in every forward)")
        if not with_box_refine or num_feature_levels != 4:
            raise NotImplementedError("monodetr_b200 implements with_box_refine=True and num_feature_levels=4 only")
        if not (isinstance(num_queries, int) and 1 <= num_queries <= MAX_QUERIES):
            raise NotImplementedError(f"num_queries={num_queries}: the device matcher takes 1 to {MAX_QUERIES} queries per group")
        self.num_queries = num_queries
        self.depthaware_transformer = depthaware_transformer
        self.depth_predictor = depth_predictor
        hidden_dim = depthaware_transformer.d_model
        self.hidden_dim = hidden_dim
        self.num_feature_levels = num_feature_levels
        self.two_stage_dino = two_stage_dino
        self.label_enc = nn.Embedding(num_classes + 1, hidden_dim - 1)
        self.class_embed = nn.Linear(hidden_dim, num_classes)
        prior_prob = 0.01
        bias_value = -math.log((1 - prior_prob) / prior_prob)
        self.class_embed.bias.data = torch.ones(num_classes) * bias_value
        self.bbox_embed = MLP(hidden_dim, hidden_dim, 6, 3)
        self.dim_embed_3d = MLP(hidden_dim, hidden_dim, 3, 2)
        self.angle_embed = MLP(hidden_dim, hidden_dim, 24, 2)
        self.depth_embed = MLP(hidden_dim, hidden_dim, 2, 2)
        self.use_dab = use_dab
        if init_box:
            nn.init.constant_(self.bbox_embed.layers[-1].weight.data, 0)
            nn.init.constant_(self.bbox_embed.layers[-1].bias.data, 0)
        if use_dab:                                 # :74-76
            self.tgt_embed = nn.Embedding(num_queries * group_num, hidden_dim)
            self.refpoint_embed = nn.Embedding(num_queries * group_num, 6)
        else:
            self.query_embed = nn.Embedding(num_queries * group_num, hidden_dim * 2)
        input_proj_list = []
        for i in range(len(backbone.strides)):
            in_channels = backbone.num_channels[i]
            input_proj_list.append(_ProjGN(nn.Conv2d(in_channels, hidden_dim, kernel_size=1), nn.GroupNorm(32, hidden_dim)))
        for _ in range(num_feature_levels - len(backbone.strides)):
            input_proj_list.append(_ProjGN(nn.Conv2d(in_channels, hidden_dim, kernel_size=3, stride=2, padding=1),
                                           nn.GroupNorm(32, hidden_dim)))
            in_channels = hidden_dim
        self.input_proj = nn.ModuleList(input_proj_list)
        self.backbone = backbone
        self.aux_loss = aux_loss
        self.with_box_refine = with_box_refine
        self.two_stage = two_stage
        self.num_classes = num_classes
        for proj in self.input_proj:
            nn.init.xavier_uniform_(proj[0].weight, gain=1)
            nn.init.constant_(proj[0].bias, 0)
        num_pred = depthaware_transformer.decoder.num_layers
        self.class_embed = _get_clones(self.class_embed, num_pred)
        self.bbox_embed = _get_clones(self.bbox_embed, num_pred)
        nn.init.constant_(self.bbox_embed[0].layers[-1].bias.data[2:], -2.0)
        self.depthaware_transformer.decoder.bbox_embed = self.bbox_embed          # alias keys (:129-131)
        self.dim_embed_3d = _get_clones(self.dim_embed_3d, num_pred)
        self.depthaware_transformer.decoder.dim_embed = self.dim_embed_3d
        self.angle_embed = _get_clones(self.angle_embed, num_pred)
        self.depth_embed = _get_clones(self.depth_embed, num_pred)

    _NO_PREPACK = ("backbone", "sa_v_proj", "query_scale", "ref_point_head", "sa_qcontent_proj", "sa_qpos_proj",
                   "sa_kcontent_proj", "sa_kpos_proj")
    # use_dab: query_scale and ref_point_head are GEMMs of every decoder layer; query_scale_bbox is never called
    _NO_PREPACK_DAB = ("backbone", "sa_v_proj", "query_scale_bbox", "sa_qcontent_proj", "sa_qpos_proj", "sa_kcontent_proj",
                       "sa_kpos_proj")

    def _gemm_weights(self):
        """Every nn.Linear / nn.Conv2d / in_proj slice the forward feeds to the tensor-core GEMMs as-is (the ResNet body
        splits its own BN-folded weights; summed decoder projections are split where they are formed)."""
        out = []
        with torch.no_grad():
            skip = self._NO_PREPACK_DAB if self.use_dab else self._NO_PREPACK
            for name, m in self.named_modules():
                if any(k in name for k in skip):
                    continue
                if isinstance(m, nn.MultiheadAttention):
                    w, c = m.in_proj_weight, m.embed_dim
                    out += [w[:c], w[c:], w[c:2 * c], w[2 * c:], w[:2 * c]]
                elif isinstance(m, (nn.Linear, nn.Conv2d)):
                    out.append(m.weight)
        return out

    def _query_embeds(self):
        """The transformer's queries (:182-199): all groups in training, the first num_queries rows in eval.  use_dab: the pair
        (tgt_embed, refpoint_embed) of weights, which the reference concatenates and the transformer splits again."""
        if self.use_dab:
            qe = (self.tgt_embed.weight, self.refpoint_embed.weight)
            return qe if self.training else tuple(w[:self.num_queries] for w in qe)
        return self.query_embed.weight if self.training else self.query_embed.weight[:self.num_queries]

    def forward(self, images, calibs, targets, img_sizes, dn_args=None):
        """images (B, 3, H, W) fp32 NCHW; calibs (B, 3, 4); targets / dn_args ignored; img_sizes (B, 2) [W, H]."""
        if self.training and images.is_cuda:
            K.begin_forward(images.device)          # new dropout masks every training forward (device-side, graph-safe)
        with tc.prepacked(self._gemm_weights() if images.is_cuda else []):
            return self._forward(images, calibs, targets, img_sizes, dn_args)

    def _forward(self, images, calibs, targets, img_sizes, dn_args=None):
        features, pos = self.backbone(images)                                      # NHWC maps, (HW, C) tables
        # The neck's projections are independent per level (the three coarse ones are tiny): the finest level stays on this
        # stream, the others run beside it.
        srcs, neck = [None] * len(features), []
        for l in range(len(features) - 1, 0, -1):
            br = Fn.Branch(15 + l, level=2)
            with br:
                srcs[l] = self.input_proj[l](features[l])
            neck.append((br, l))
        extra = None
        if self.num_feature_levels == len(features) + 1:
            extra = Fn.Branch(15, level=2)
            with extra:
                src_extra = self.input_proj[len(features)](features[-1])
        srcs[0] = self.input_proj[0](features[0])
        for br, l in neck:
            br.join(srcs[l])
        if extra is not None:
            extra.join(src_extra)
            srcs.append(src_extra)
            pos.append(self.backbone[1](src_extra))
        for l in range(len(srcs), self.num_feature_levels):
            src = self.input_proj[l](features[-1] if l == len(features) else srcs[-1])
            srcs.append(src)
            pos.append(self.backbone[1](src))
        query_embeds = self._query_embeds()

        # The depth predictor and the visual encoder both depend on `srcs` only: the (small) depth branch runs on its own
        # stream beside the encoder and is joined right before the decoder, its first consumer.
        depth_branch = Fn.Branch(0)
        with depth_branch:
            depth_logits, depth_pos_embed, weighted_depth, depth_pos_embed_ip = self.depth_predictor(srcs, None, pos[1])
        hs, init_reference, inter_references, inter_references_dim, boxes = self.depthaware_transformer(
            srcs, None, pos, query_embeds, depth_pos_embed, depth_pos_embed_ip,
            before_decoder=lambda: depth_branch.join(depth_logits, depth_pos_embed, weighted_depth, depth_pos_embed_ip))

        outputs_coords, outputs_classes, outputs_3d_dims, outputs_depths, outputs_angles = [], [], [], [], []
        branches = []
        for lvl in range(hs.shape[0]):
            # The heads of the three decoder levels are independent chains of small GEMMs (launch-latency bound): one stream each.
            br = Fn.Branch(head_stream(lvl))
            with br:
                # The reference re-evaluates bbox_embed[lvl](hs[lvl]) + inverse_sigmoid(reference) here (:216-228); that is the
                # very tensor the decoder already formed before detaching it, so it is reused (same values, same gradients).
                outputs_coord = boxes[lvl]
                outputs_coords.append(outputs_coord)
                cls = self.class_embed[lvl]
                outputs_classes.append(Fn.linear(hs[lvl], cls.weight, cls.bias))
                size3d = inter_references_dim[lvl]
                outputs_3d_dims.append(size3d)
                depth_reg = self.depth_embed[lvl](hs[lvl])
                # regressed + geometric + depth-map depth, averaged (:230-262; the sample grid uses detached centres): one kernel
                depth_ave = Fn.head_depth(outputs_coord, size3d, depth_reg, weighted_depth, calibs, img_sizes)
                outputs_depths.append(depth_ave)
                outputs_angles.append(self.angle_embed[lvl](hs[lvl]))
            branches.append(br)
        for lvl, br in enumerate(branches):
            br.join(outputs_classes[lvl], outputs_depths[lvl], outputs_angles[lvl])

        out = {"pred_logits": outputs_classes[-1], "pred_boxes": outputs_coords[-1], "pred_3d_dim": outputs_3d_dims[-1],
               "pred_depth": outputs_depths[-1], "pred_angle": outputs_angles[-1],
               "pred_depth_map_logits": depth_logits.permute(0, 3, 1, 2)}          # (B, 81, H, W) view of the NHWC logits
        if self.aux_loss:
            out["aux_outputs"] = [{"pred_logits": a, "pred_boxes": b, "pred_3d_dim": c, "pred_angle": d, "pred_depth": e}
                                  for a, b, c, d, e in zip(outputs_classes[:-1], outputs_coords[:-1], outputs_3d_dims[:-1],
                                                           outputs_angles[:-1], outputs_depths[:-1])]
        return out


def _reference_criterion(cfg):
    """SetCriterion + HungarianMatcher exactly as the reference's build() assembles them (monodetr.py:578-612), taken from
    the reference package when it is importable (`lib.models.monodetr` on PYTHONPATH, as under tools/train_val.py).  The
    criterion sits AFTER the hot path (SURVEY.md 8f-1) and is used unchanged; returns None when the package is absent."""
    try:
        from lib.models.monodetr.matcher import build_matcher
        from lib.models.monodetr.monodetr import SetCriterion
    except Exception:          # not installed / not importable on this torch: the caller gets (model, None)
        return None
    matcher = build_matcher(cfg)
    weight_dict = {"loss_ce": cfg["cls_loss_coef"], "loss_bbox": cfg["bbox_loss_coef"], "loss_giou": cfg["giou_loss_coef"],
                   "loss_dim": cfg["dim_loss_coef"], "loss_angle": cfg["angle_loss_coef"], "loss_depth": cfg["depth_loss_coef"],
                   "loss_center": cfg["3dcenter_loss_coef"], "loss_depth_map": cfg["depth_map_loss_coef"]}
    if cfg.get("use_dn"):
        weight_dict.update({"tgt_loss_ce": cfg["cls_loss_coef"], "tgt_loss_bbox": cfg["bbox_loss_coef"],
                            "tgt_loss_giou": cfg["giou_loss_coef"], "tgt_loss_angle": cfg["angle_loss_coef"],
                            "tgt_loss_center": cfg["3dcenter_loss_coef"]})
    if cfg["aux_loss"]:
        aux = {}
        for i in range(cfg["dec_layers"] - 1):
            aux.update({k + f"_{i}": v for k, v in weight_dict.items()})
        aux.update({k + "_enc": v for k, v in weight_dict.items()})
        weight_dict.update(aux)
    losses = ["labels", "boxes", "cardinality", "depths", "dims", "angles", "center", "depth_map"]
    criterion = SetCriterion(cfg["num_classes"], matcher=matcher, weight_dict=weight_dict, focal_alpha=cfg["focal_alpha"],
                             losses=losses)
    return criterion.to(torch.device(cfg["device"]))


def build(cfg, criterion_builder=None):
    """Same contract as the reference's build(cfg) (:550-614): returns (model, criterion).  The criterion (SetCriterion +
    HungarianMatcher) is the step after the hot path (SURVEY.md 8f-1): `criterion_builder(cfg)` if given; else, for a cfg
    that carries the loss weights, the reference's own classes when `lib.models.monodetr` is importable (the situation
    inside tools/train_val.py) unless cfg["criterion"] == "device", and otherwise this package's device-resident criterion
    (monodetr_b200.criterion: same keys / values / gradients, no host synchronisation); None for a cfg without loss weights."""
    backbone = build_backbone(cfg)
    depthaware_transformer = build_depthaware_transformer(cfg)
    depth_predictor = DepthPredictor(cfg)
    model = MonoDETR(backbone, depthaware_transformer, depth_predictor, num_classes=cfg["num_classes"],
                     num_queries=cfg["num_queries"], aux_loss=cfg["aux_loss"], num_feature_levels=cfg["num_feature_levels"],
                     with_box_refine=cfg["with_box_refine"], two_stage=cfg["two_stage"], init_box=cfg["init_box"],
                     use_dab=cfg["use_dab"], two_stage_dino=cfg["two_stage_dino"])
    if criterion_builder is not None:
        criterion = criterion_builder(cfg)
    elif "cls_loss_coef" in cfg:                   # a full configs/monodetr.yaml model section (loss weights present)
        criterion = None if cfg.get("criterion") == "device" else _reference_criterion(cfg)
        if criterion is None:
            from .criterion import build_criterion
            criterion = build_criterion(cfg).to(torch.device(cfg["device"]))
    else:
        criterion = None
    return model, criterion


DEFAULT_MODEL_CFG = {
    # configs/monodetr.yaml `model:` section (the keys the builders read, SURVEY.md 5)
    "num_classes": 3, "return_intermediate_dec": True, "device": "cuda", "backbone": "resnet50", "train_backbone": True,
    "num_feature_levels": 4, "dilation": False, "position_embedding": "sine", "masks": False, "mode": "LID",
    "num_depth_bins": 80, "depth_min": 1e-3, "depth_max": 60.0, "with_box_refine": True, "two_stage": False,
    "use_dab": False, "use_dn": False, "two_stage_dino": False, "init_box": False, "enc_layers": 3, "dec_layers": 3,
    "hidden_dim": 256, "dim_feedforward": 256, "dropout": 0.1, "nheads": 8, "num_queries": 50, "enc_n_points": 4,
    "dec_n_points": 4, "aux_loss": True,
}
