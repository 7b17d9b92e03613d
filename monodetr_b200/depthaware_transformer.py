"""Depth-aware transformer -- mirror of lib/models/monodetr/depthaware_transformer.py (DepthAwareTransformer
:69-312, VisualEncoderLayer/VisualEncoder :315-384, DepthAwareDecoderLayer :387-515, DepthAwareDecoder :518-626,
build_depthaware_transformer :644-660; the configs/monodetr.yaml branch and the anchor-box query branch use_dab; two_stage /
two_stage_dino raise) with identical parameter names, running on the sm_90a kernels.

Tensors are batch-first and token-major ((B, L, C)); feature levels arrive NHWC so flattening is a view.
"""
import copy

import torch
from torch import nn
from torch.nn.init import constant_, normal_, xavier_uniform_

from . import functional as Fn
from .ms_deform_attn import MSDeformAttn


def inverse_sigmoid(x, eps=1e-5):      # utils/misc.py:473-477
    x = x.clamp(min=0, max=1)
    x1 = x.clamp(min=eps)
    x2 = (1 - x).clamp(min=eps)
    return torch.log(x1 / x2)


class MLP(nn.Module):
    """Very simple multi-layer perceptron (reference :14-27)."""

    def __init__(self, input_dim, hidden_dim, output_dim, num_layers):
        super().__init__()
        self.num_layers = num_layers
        h = [hidden_dim] * (num_layers - 1)
        self.layers = nn.ModuleList(nn.Linear(n, k) for n, k in zip([input_dim] + h, h + [output_dim]))

    def forward(self, x):
        for i, layer in enumerate(self.layers):
            x = Fn.linear(x, layer.weight, layer.bias, relu=(i < self.num_layers - 1))
        return x


def _get_clones(module, N):
    return nn.ModuleList([copy.deepcopy(module) for _ in range(N)])


class VisualEncoderLayer(nn.Module):
    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4):
        super().__init__()
        self.self_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.dropout2 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.dropout3 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(d_model)
        self.site_base = 0

    def forward(self, src, pos, reference_points, spatial_shapes, level_start_index, padding_mask=None):
        sb = self.site_base
        if (self.dropout1.p == self.dropout2.p == self.dropout3.p and pos is not None
                and Fn.encoder_layer_fusable(self, src, reference_points, padding_mask)):
            return Fn.encoder_layer(self, src, pos, reference_points, spatial_shapes, level_start_index)   # one autograd node
        src2 = self.self_attn(src + pos, reference_points, src, spatial_shapes, level_start_index, padding_mask)
        src = Fn.add_layernorm(src, src2, self.norm1.weight, self.norm1.bias, self.norm1.eps, self.dropout1.p, self.training, sb)
        h = Fn.linear(src, self.linear1.weight, self.linear1.bias, relu=True)
        h = Fn.dropout(h, self.dropout2.p, self.training, sb + 1)
        src2 = Fn.linear(h, self.linear2.weight, self.linear2.bias)
        return Fn.add_layernorm(src, src2, self.norm2.weight, self.norm2.bias, self.norm2.eps, self.dropout3.p, self.training, sb + 2)


class VisualEncoder(nn.Module):
    def __init__(self, encoder_layer, num_layers):
        super().__init__()
        self.layers = _get_clones(encoder_layer, num_layers)
        for i, l in enumerate(self.layers):
            l.site_base = 100 + 10 * i
        self.num_layers = num_layers
        self._ref_cache = {}

    def get_reference_points(self, shapes, B, device):
        """reference :363-376 with valid_ratios == 1 (masks are all-False on this path): pixel centres, input-independent."""
        key = (tuple(shapes), str(device))
        if key not in self._ref_cache:
            pts = []
            for (H_, W_) in shapes:
                ref_y, ref_x = torch.meshgrid(torch.linspace(0.5, H_ - 0.5, H_, dtype=torch.float32, device=device),
                                              torch.linspace(0.5, W_ - 0.5, W_, dtype=torch.float32, device=device), indexing="ij")
                pts.append(torch.stack((ref_x.reshape(-1) / W_, ref_y.reshape(-1) / H_), -1))
            ref = torch.cat(pts, 0)
            self._ref_cache[key] = ref[:, None].expand(-1, len(shapes), -1).contiguous()     # (S, L, 2)
        return self._ref_cache[key][None].expand(B, -1, -1, -1)

    def forward(self, src, shapes, spatial_shapes, level_start_index, pos=None, padding_mask=None):
        reference_points = self.get_reference_points(shapes, src.shape[0], src.device)
        output = src
        for layer in self.layers:
            output = layer(output, pos, reference_points, spatial_shapes, level_start_index, padding_mask)
        return output


class DepthAwareDecoderLayer(nn.Module):
    def __init__(self, d_model=256, d_ffn=1024, dropout=0.1, activation="relu", n_levels=4, n_heads=8, n_points=4, group_num=1):
        super().__init__()
        self.cross_attn = MSDeformAttn(d_model, n_levels, n_heads, n_points)
        self.dropout1 = nn.Dropout(dropout)
        self.norm1 = nn.LayerNorm(d_model)
        self.cross_attn_depth = nn.MultiheadAttention(d_model, n_heads, dropout=dropout)    # parameter containers
        self.dropout_depth = nn.Dropout(dropout)
        self.norm_depth = nn.LayerNorm(d_model)
        self.self_attn = nn.MultiheadAttention(d_model, n_heads, dropout=dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.norm2 = nn.LayerNorm(d_model)
        self.linear1 = nn.Linear(d_model, d_ffn)
        self.dropout3 = nn.Dropout(dropout)
        self.linear2 = nn.Linear(d_ffn, d_model)
        self.dropout4 = nn.Dropout(dropout)
        self.norm3 = nn.LayerNorm(d_model)
        self.group_num = group_num
        self.sa_qcontent_proj = nn.Linear(d_model, d_model)
        self.sa_qpos_proj = nn.Linear(d_model, d_model)
        self.sa_kcontent_proj = nn.Linear(d_model, d_model)
        self.sa_kpos_proj = nn.Linear(d_model, d_model)
        self.sa_v_proj = nn.Linear(d_model, d_model)     # kept for state_dict parity; its output is discarded (:471,477)
        self.nhead = n_heads
        self.site_base = 0

    def depth_kv(self, depth_pos_embed):
        """Key / value projection of the depth cross attention (one GEMM): a function of the depth embedding only."""
        a = self.cross_attn_depth
        c = a.embed_dim
        return Fn.linear(depth_pos_embed, a.in_proj_weight[c:], a.in_proj_bias[c:])

    def forward(self, tgt, query_pos, reference_points, src, src_spatial_shapes, level_start_index, src_padding_mask,
                depth_pos_embed, mask_depth, bs, ahead=None):
        """tgt/query_pos (B, nq, C); src (B, S, C); depth_pos_embed (B, 1920, C) batch-first.
        `ahead`: optional dict of work the decoder started on branch streams -- "kv" / "value" (callables returning the depth
        key-value projection / the projected memory once joined) and "reference_points" (callable returning the boxes of the
        previous layer, needed only by the deformable cross attention)."""
        sb = self.site_base
        c = tgt.shape[-1]
        B, nq, _ = tgt.shape
        ahead = ahead or {}
        # ---- depth cross attention (:456-462): q = tgt (no positional term), k = v = depth_pos_embed -------------
        a = self.cross_attn_depth
        q = Fn.linear(tgt, a.in_proj_weight[:c], a.in_proj_bias[:c])
        kv = ahead["kv"]() if "kv" in ahead else self.depth_kv(depth_pos_embed)                     # fused k,v projection
        o = Fn.attention(q, kv[..., :c], kv[..., c:], mask_depth, a.dropout, self.training, sb, self.nhead)
        tgt2 = Fn.linear(o, a.out_proj.weight, a.out_proj.bias)
        tgt = Fn.add_layernorm(tgt, tgt2, self.norm_depth.weight, self.norm_depth.bias, self.norm_depth.eps,
                               self.dropout_depth.p, self.training, sb + 1)
        # ---- (group-wise) self attention (:465-503) ------------------------------------------------------------------
        qk = tgt + query_pos
        # q_content + q_pos are two linears of the SAME input: one GEMM with the summed weights (:467-473)
        s = self.self_attn
        # the key chain and the value projection do not depend on the query chain: three streams, two GEMMs deep instead of five
        br_k, br_v = Fn.Branch(7, level=2), Fn.Branch(8, level=2)
        with br_k:
            ks = Fn.linear(qk, self.sa_kcontent_proj.weight + self.sa_kpos_proj.weight, self.sa_kcontent_proj.bias + self.sa_kpos_proj.bias)
            k = Fn.linear(ks, s.in_proj_weight[c:2 * c], s.in_proj_bias[c:2 * c])
        with br_v:
            v = Fn.linear(tgt, s.in_proj_weight[2 * c:], s.in_proj_bias[2 * c:])                      # v = tgt (:477)
        qs = Fn.linear(qk, self.sa_qcontent_proj.weight + self.sa_qpos_proj.weight, self.sa_qcontent_proj.bias + self.sa_qpos_proj.bias)
        q = Fn.linear(qs, s.in_proj_weight[:c], s.in_proj_bias[:c])
        br_k.join(k)
        br_v.join(v)
        if self.training:
            # 11 groups of 50 queries attend only within their group (:480-494): fold groups into the batch (a view)
            g = self.group_num
            per = nq // g
            o = Fn.attention(q.reshape(B * g, per, c), k.reshape(B * g, per, c), v.reshape(B * g, per, c), None,
                             s.dropout, True, sb + 2, self.nhead).reshape(B, nq, c)
        else:
            o = Fn.attention(q, k, v, None, 0.0, False, sb + 2, self.nhead)
        tgt2 = Fn.linear(o, s.out_proj.weight, s.out_proj.bias)
        tgt = Fn.add_layernorm(tgt, tgt2, self.norm2.weight, self.norm2.bias, self.norm2.eps, self.dropout2.p, self.training, sb + 3)
        # ---- deformable cross attention over the image memory (:506-510) ---------------------------------------------
        if "reference_points" in ahead:
            reference_points = ahead["reference_points"]()
        tgt2 = self.cross_attn(tgt + query_pos, reference_points, src, src_spatial_shapes, level_start_index, src_padding_mask,
                               value=ahead["value"]() if "value" in ahead else None)
        tgt = Fn.add_layernorm(tgt, tgt2, self.norm1.weight, self.norm1.bias, self.norm1.eps, self.dropout1.p, self.training, sb + 4)
        # ---- ffn (:431-435) ----------------------------------------------------------------------------------------------
        h = Fn.linear(tgt, self.linear1.weight, self.linear1.bias, relu=True)
        h = Fn.dropout(h, self.dropout3.p, self.training, sb + 5)
        tgt2 = Fn.linear(h, self.linear2.weight, self.linear2.bias)
        return Fn.add_layernorm(tgt, tgt2, self.norm3.weight, self.norm3.bias, self.norm3.eps, self.dropout4.p, self.training, sb + 6)


def ahead_streams(lid):
    """Branch stream indices of decoder layer `lid`'s ahead-of-time depth key-value and value projections.  Layers 0-2 keep
    9-11 / 12-14; deeper layers take 19 and up, clear of the neck's 15-18 and of the heads' (MonoDETR._forward)."""
    return (9 + lid, 12 + lid) if lid < 3 else (19 + 2 * (lid - 3), 20 + 2 * (lid - 3))


class DepthAwareDecoder(nn.Module):
    def __init__(self, decoder_layer, num_layers, return_intermediate=False, d_model=None, use_dab=False):
        super().__init__()
        self.layers = _get_clones(decoder_layer, num_layers)
        for i, l in enumerate(self.layers):
            l.site_base = 200 + 10 * i
        self.num_layers = num_layers
        self.return_intermediate = return_intermediate
        self.bbox_embed = None
        self.dim_embed = None
        self.class_embed = None
        self.use_dab = use_dab
        if use_dab:                             # :530-533; query_scale_bbox is never called by the reference
            self.query_scale = MLP(d_model, d_model, d_model, 2)
            self.query_scale_bbox = MLP(d_model, 2, 2, 2)
            self.ref_point_head = MLP(3 * d_model, d_model, d_model, 2)
        else:
            # unused on the default path but part of the reference state_dict (:541-542)
            self.query_scale = MLP(d_model, d_model, d_model, 2)
            self.ref_point_head = MLP(d_model, d_model, 2, 2)

    def forward(self, tgt, reference_points, src, src_spatial_shapes, src_level_start_index, query_pos=None,
                src_padding_mask=None, depth_pos_embed=None, mask_depth=None, bs=None):
        """Returns stacked (hs, references (undetached sigmoid boxes), dims) -- see note in MonoDETR.forward.
        use_dab: `reference_points` is Fn.anchors' (sine, msda, head) triple of the anchors and `query_pos` is None; each layer
        forms its own query position from its boxes (:584-588)."""
        output = tgt
        raw_pos = None
        if self.use_dab:
            # layer 0's boxes are the anchors, the same for every image: sine embedding and ref_point_head on nq rows
            r_sine, r_msda, reference_points = reference_points
            raw_pos = self.ref_point_head(Fn.sine_embed(r_sine))
        n_levels = src_spatial_shapes.shape[0]
        intermediate, intermediate_boxes, intermediate_refs, intermediate_dims = [], [], [], []
        # Work that depends on the memory / the depth embedding only is started now on branch streams and joined where each layer
        # first needs it: the depth key-value projections (3 GEMMs) and the deformable attention's value projections (3 large
        # GEMMs that fill the SMs the decoder's small launches leave idle).
        ahead_kv, ahead_val = [], []
        for lid, layer in enumerate(self.layers):
            bk, bv = (Fn.Branch(i, level=2) for i in ahead_streams(lid))
            with bk:
                kv = layer.depth_kv(depth_pos_embed)
            with bv:
                val = layer.cross_attn.project_value(src, src_padding_mask)
            ahead_kv.append((bk, kv))
            ahead_val.append((bv, val))

        def joined(pair):
            def get():
                pair[0].join(pair[1])
                return pair[1]
            return get

        box_branch = None                       # (branch, boxes) of the previous layer: joined right before its first use
        dim_branches = []
        for lid, layer in enumerate(self.layers):
            ahead = {"kv": joined(ahead_kv[lid]), "value": joined(ahead_val[lid])}
            if self.use_dab:
                if box_branch is None:
                    query_pos = Fn.query_pos(None, raw_pos, output.shape[0])           # pos_scale = 1 at layer 0
                else:
                    box_branch[0].join(box_branch[1])                              # this layer's position needs its boxes first
                    raw_pos = self.ref_point_head(Fn.sine_embed(box_branch[1].detach()))
                    query_pos = Fn.query_pos(self.query_scale(output), raw_pos, output.shape[0])
            if box_branch is None:
                if self.use_dab:
                    ref_in = r_msda                                                 # (nq, 6): shared by the batch and the levels
                else:
                    ref_in = reference_points[:, :, None].expand(-1, -1, n_levels, -1)   # valid_ratios == 1 (:565-571): broadcast over levels
            else:
                ref_in = None
                ahead["reference_points"] = (lambda bb: lambda: (bb[0].join(bb[1]), bb[1].detach()[:, :, None].expand(-1, -1, n_levels, -1))[1])(box_branch)
            output = layer(output, query_pos, ref_in, src, src_spatial_shapes, src_level_start_index,
                           src_padding_mask, depth_pos_embed, mask_depth, bs, ahead=ahead)
            if box_branch is not None:
                reference_points = box_branch[1].detach()                       # (joined inside the layer)
                intermediate_refs.append(reference_points)
            # box refinement (:602-613) and the size head read this layer's output but the next layer needs the boxes only at its
            # deformable cross attention: both leave the critical path
            bb = Fn.Branch(5, level=2)
            with bb:
                tmp = self.bbox_embed[lid](output)
                # (tmp + inverse_sigmoid(ref)).sigmoid() on the first 2 / all 6 components: one fused kernel
                new_reference_points = Fn.box_refine(tmp, reference_points)
            box_branch = (bb, new_reference_points)
            bd = Fn.Branch(6, level=2)
            with bd:
                reference_dims = self.dim_embed[lid](output)
            dim_branches.append((bd, reference_dims))
            intermediate_boxes.append(new_reference_points)                     # with gradient: == outputs_coord of monodetr.py:216-228
            intermediate.append(output)
            intermediate_dims.append(reference_dims)
        box_branch[0].join(box_branch[1])
        intermediate_refs.append(box_branch[1].detach())
        for bd, dims in dim_branches:
            bd.join(dims)
        return torch.stack(intermediate), torch.stack(intermediate_refs), torch.stack(intermediate_dims), intermediate_boxes


SUPPORTED_HEAD_DIMS = (16, 32, 64)       # head widths csrc/attention.cu is compiled for
SUPPORTED_POINTS = range(1, 9)           # sampling points per level: 2, 4 and 8 on the fused kernels, the rest on the two-step path
# Encoder / decoder depth: the device criterion takes at most 6 decoder layers (MDB_CRITERION_MAX_LAYERS).  Up to 6 layers the
# dropout sites of the encoder (100 + 10 i + 0..2) and the decoder (200 + 10 i + 0..6) stay below 160 and 260: none collide.
SUPPORTED_LAYERS = range(1, 7)


class DepthAwareTransformer(nn.Module):
    def __init__(self, d_model=256, nhead=8, num_encoder_layers=6, num_decoder_layers=6, dim_feedforward=1024, dropout=0.1,
                 activation="relu", return_intermediate_dec=False, num_feature_levels=4, dec_n_points=4, enc_n_points=4,
                 two_stage=False, two_stage_num_proposals=50, group_num=11, use_dab=False, two_stage_dino=False):
        super().__init__()
        if two_stage or two_stage_dino:
            raise NotImplementedError("two_stage / two_stage_dino are not implemented: the reference itself fails with them "
                                      "(two_stage in the training forward, two_stage_dino in every forward)")
        if d_model % nhead or d_model // nhead not in SUPPORTED_HEAD_DIMS:
            supported = ", ".join(str(d_model // hd) for hd in sorted(SUPPORTED_HEAD_DIMS, reverse=True))
            raise NotImplementedError(f"nheads={nhead} at hidden_dim={d_model}: the attention kernels take head widths "
                                      f"{sorted(SUPPORTED_HEAD_DIMS)}, so nheads must be one of {supported}")
        for name, n in (("enc_n_points", enc_n_points), ("dec_n_points", dec_n_points)):
            if not (isinstance(n, int) and n in SUPPORTED_POINTS):
                raise NotImplementedError(f"{name}={n}: the deformable-attention kernels take {SUPPORTED_POINTS[0]} to "
                                          f"{SUPPORTED_POINTS[-1]} sampling points per level")
        for name, n in (("enc_layers", num_encoder_layers), ("dec_layers", num_decoder_layers)):
            if not (isinstance(n, int) and n in SUPPORTED_LAYERS):
                raise NotImplementedError(f"{name}={n}: {SUPPORTED_LAYERS[0]} to {SUPPORTED_LAYERS[-1]} layers are implemented")
        if not (isinstance(dim_feedforward, int) and dim_feedforward > 0 and dim_feedforward % 4 == 0):
            raise NotImplementedError(f"dim_feedforward={dim_feedforward}: a positive multiple of 4 is implemented")
        if not return_intermediate_dec:
            raise NotImplementedError("return_intermediate_dec=False is not implemented: the reference itself fails with it (its "
                                      "decoder then returns two values where the transformer unpacks three)")
        if d_model != 256:
            raise NotImplementedError(f"hidden_dim={d_model} is not implemented: the reference itself fails with it (its "
                                      "depth_pos_embed is 256 wide and is added to a hidden_dim-wide tensor)")
        self.d_model, self.nhead, self.group_num = d_model, nhead, group_num
        self.two_stage, self.use_dab, self.two_stage_dino = two_stage, use_dab, two_stage_dino
        self.two_stage_num_proposals = two_stage_num_proposals
        encoder_layer = VisualEncoderLayer(d_model, dim_feedforward, dropout, activation, num_feature_levels, nhead, enc_n_points)
        self.encoder = VisualEncoder(encoder_layer, num_encoder_layers)
        decoder_layer = DepthAwareDecoderLayer(d_model, dim_feedforward, dropout, activation, num_feature_levels, nhead,
                                               dec_n_points, group_num=group_num)
        self.decoder = DepthAwareDecoder(decoder_layer, num_decoder_layers, return_intermediate_dec, d_model, use_dab=use_dab)
        self.level_embed = nn.Parameter(torch.Tensor(num_feature_levels, d_model))
        if not use_dab:
            self.reference_points = nn.Linear(d_model, 2)
        self._reset_parameters()

    def _reset_parameters(self):
        for p in self.parameters():
            if p.dim() > 1:
                nn.init.xavier_uniform_(p)
        for m in self.modules():
            if isinstance(m, MSDeformAttn):
                m._reset_parameters()
        if not self.use_dab:
            xavier_uniform_(self.reference_points.weight.data, gain=1.0)
            constant_(self.reference_points.bias.data, 0.)
        normal_(self.level_embed)

    def _shape_tensors(self, shapes, dev):
        """int64 (L,2) shapes and (L,) level starts on the device, cached (no host->device copy per step; graph-safe)."""
        key = (tuple(shapes), str(dev))
        cache = self.__dict__.setdefault("_shape_cache", {})
        if key not in cache:
            ss = torch.as_tensor(shapes, dtype=torch.long, device=dev)
            cache[key] = (ss, torch.cat((ss.new_zeros((1,)), ss.prod(1).cumsum(0)[:-1])))
        return cache[key]

    def forward(self, srcs, masks, pos_embeds, query_embed=None, depth_pos_embed=None, depth_pos_embed_ip=None, attn_mask=None,
                before_decoder=None):
        """srcs: list of NHWC maps (B, H_l, W_l, C); masks: None (all-False) or list of (B, H_l, W_l) bool;
        pos_embeds: list of (H_l*W_l, C); query_embed (nq, 2C), or with use_dab the pair (tgt (nq, C), anchors (nq, 6)) of
        unactivated embeddings; depth_pos_embed (B, HW1, C).
        Returns hs (L, B, nq, C), init_reference (B, nq, 2), inter_references (L, B, nq, 6), inter_dims (L, B, nq, 3),
        plus the undetached per-layer boxes (list) used by MonoDETR.forward."""
        assert query_embed is not None
        B = srcs[0].shape[0]
        dev = srcs[0].device
        shapes = [tuple(s.shape[1:3]) for s in srcs]
        src_flatten = torch.cat([s.reshape(B, -1, s.shape[-1]) for s in srcs], 1)
        lvl_pos = torch.cat([pe + self.level_embed[l].view(1, -1) for l, pe in enumerate(pos_embeds)], 0)   # (S, C)
        mask_flatten = None
        if masks is not None and any(m is not None and bool(m.any()) for m in masks):
            raise NotImplementedError("padding masks: this path always has all-False masks (backbone.py:88)")
        spatial_shapes, level_start_index = self._shape_tensors(shapes, dev)
        memory = self.encoder(src_flatten, shapes, spatial_shapes, level_start_index, lvl_pos, mask_flatten)
        c = memory.shape[-1]
        if self.use_dab:                         # :255-260 (the decoder repeats the boxes over the batch, :557-558)
            tgt, refanchor = query_embed
            tgt = tgt.unsqueeze(0).expand(B, -1, -1).contiguous()
            query_pos = None
            reference_points = Fn.anchors(refanchor, B)
            init_reference_out = reference_points[2]
        else:
            query_pos, tgt = torch.split(query_embed, c, dim=1)
            query_pos = query_pos.unsqueeze(0).expand(B, -1, -1)
            tgt = tgt.unsqueeze(0).expand(B, -1, -1).contiguous()
            reference_points = Fn.linear(query_pos.contiguous(), self.reference_points.weight, self.reference_points.bias).sigmoid()
            init_reference_out = reference_points
        if before_decoder is not None:           # (the depth predictor may still be running on its own stream: join it here)
            before_decoder()
        hs, inter_references, inter_dims, boxes = self.decoder(tgt, reference_points, memory, spatial_shapes, level_start_index,
                                                              query_pos, mask_flatten, depth_pos_embed, None, bs=B)
        return hs, init_reference_out, inter_references, inter_dims, boxes


def build_depthaware_transformer(cfg):
    return DepthAwareTransformer(
        d_model=cfg["hidden_dim"], dropout=cfg["dropout"], activation="relu", nhead=cfg["nheads"],
        dim_feedforward=cfg["dim_feedforward"], num_encoder_layers=cfg["enc_layers"], num_decoder_layers=cfg["dec_layers"],
        return_intermediate_dec=cfg["return_intermediate_dec"], num_feature_levels=cfg["num_feature_levels"],
        dec_n_points=cfg["dec_n_points"], enc_n_points=cfg["enc_n_points"], two_stage=cfg["two_stage"],
        two_stage_num_proposals=cfg["num_queries"], use_dab=cfg["use_dab"], two_stage_dino=cfg["two_stage_dino"])
