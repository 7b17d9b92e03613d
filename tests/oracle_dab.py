"""TEST INFRASTRUCTURE: the CPU oracle (oracle/monodetr_torch.py) for the anchor-box query branch (`use_dab: True`).

oracle/monodetr_torch.py states the default branch; this module restates only what use_dab changes -- the state_dict entries
(tgt_embed / refpoint_embed instead of query_embed, no transformer reference_points, the decoder's DAB MLPs) and the transformer
(depthaware_transformer.py:255-260, :557-599: per-layer sine query positions from the current boxes, layer 0 on the anchors
sigmoid(refpoint_embed)) -- and runs everything else through that module's own functions.  Pinned to the unmodified reference
by tests/test_oracle_dab.py (tests/golden/dab.npz)."""
import math

import torch
import torch.nn.functional as F

from oracle import monodetr_torch as om

CFG = dict(om.CFG, use_dab=True)
_default_spec = om.state_dict_spec


def gen_sineembed_for_position(pos):
    """depthaware_transformer.py:29-65, 6-d case: (..., 6) -> (..., 768) = [y | x | l | r | t | b]."""
    scale = 2 * math.pi
    dim_t = torch.arange(128, dtype=torch.float32, device=pos.device)
    dim_t = 10000 ** (2 * (dim_t // 2) / 128)
    out = []
    for i in (1, 0, 2, 3, 4, 5):
        p = pos[..., i] * scale
        p = p[..., None] / dim_t
        out.append(torch.stack((p[..., 0::2].sin(), p[..., 1::2].cos()), dim=-1).flatten(-2))
    return torch.cat(out, -1)


def state_dict_spec(cfg=CFG, base_spec=None):
    """The default spec (or `base_spec`, e.g. another backbone's) with the use_dab entries, in the reference's order."""
    c = cfg["hidden_dim"]
    nq = cfg["num_queries"] * cfg["group_num"]
    t = "depthaware_transformer."
    spec = {}
    for k, v in (base_spec if base_spec is not None else _default_spec(cfg)).items():
        if k == "query_embed.weight":
            spec["tgt_embed.weight"] = (nq, c)
            spec["refpoint_embed.weight"] = (nq, 6)
        elif k.startswith(t + "reference_points.") or k.startswith(t + "decoder.query_scale.") \
                or k.startswith(t + "decoder.ref_point_head."):
            continue
        else:
            spec[k] = v
    for p, dims in (("query_scale", (c, c, c)), ("query_scale_bbox", (c, 2, 2)), ("ref_point_head", (3 * c, c, c))):
        spec[f"{t}decoder.{p}.layers.0.weight"] = (dims[1], dims[0]); spec[f"{t}decoder.{p}.layers.0.bias"] = (dims[1],)
        spec[f"{t}decoder.{p}.layers.1.weight"] = (dims[2], dims[1]); spec[f"{t}decoder.{p}.layers.1.bias"] = (dims[2],)
    return spec


def transformer(sd, srcs, pos_embeds, query_embed, depth_pos_embed, training, cfg=CFG):
    """depthaware_transformer.py:199-312 with use_dab; query_embed = cat(tgt_embed, refpoint_embed) rows (monodetr.py:182-191)."""
    p = "depthaware_transformer."
    B = srcs[0].shape[0]
    dev = srcs[0].device
    shapes = [tuple(s.shape[-2:]) for s in srcs]
    src_flatten = torch.cat([s.flatten(2).transpose(1, 2) for s in srcs], 1)
    lvl_pos = torch.cat([pe.flatten(2).transpose(1, 2) + sd[p + "level_embed"][l].view(1, 1, -1)
                         for l, pe in enumerate(pos_embeds)], 1)
    spatial_shapes = torch.as_tensor(shapes, dtype=torch.long, device=dev)
    ref_enc = om.encoder_reference_points(shapes, B, dev)
    memory = src_flatten
    for l in range(cfg["enc_layers"]):
        e = f"{p}encoder.layers.{l}"
        src2 = om.ms_deform_attn(sd, e + ".self_attn", memory + lvl_pos, ref_enc, memory, spatial_shapes)
        memory = om.layer_norm(sd, e + ".norm1", memory + om._drop(src2))
        memory = om.layer_norm(sd, e + ".norm2", memory + om._drop(om.linear(sd, e + ".linear2",
                                                                            om._drop(F.relu(om.linear(sd, e + ".linear1", memory))))))
    c = memory.shape[-1]
    init_reference = query_embed[..., c:].sigmoid()                 # :255-260, (nq, 6)
    tgt = query_embed[..., :c].unsqueeze(0).expand(B, -1, -1)
    reference_points = init_reference[None].repeat(B, 1, 1)         # :557-558
    dpe = depth_pos_embed.flatten(2).permute(2, 0, 1)
    output = tgt
    G = cfg["group_num"]
    inter, inter_ref, inter_dim = [], [], []
    for l in range(cfg["dec_layers"]):                              # :563-613
        d = f"{p}decoder.layers.{l}"
        ref_in = reference_points[:, :, None].expand(-1, -1, len(shapes), -1)
        raw = om.mlp(sd, p + "decoder.ref_point_head", gen_sineembed_for_position(ref_in[:, :, 0, :]), 2)
        query_pos = raw if l == 0 else om.mlp(sd, p + "decoder.query_scale", output, 2) * raw
        tgt2 = om.mha(sd, d + ".cross_attn_depth", output.transpose(0, 1), dpe, dpe).transpose(0, 1)
        t = om.layer_norm(sd, d + ".norm_depth", output + om._drop(tgt2))
        qk = t + query_pos
        q = (om.linear(sd, d + ".sa_qcontent_proj", qk) + om.linear(sd, d + ".sa_qpos_proj", qk)).transpose(0, 1)
        k = (om.linear(sd, d + ".sa_kcontent_proj", qk) + om.linear(sd, d + ".sa_kpos_proj", qk)).transpose(0, 1)
        v = t.transpose(0, 1)
        nq = q.shape[0]
        if training:
            q = torch.cat(q.split(nq // G, dim=0), dim=1)
            k = torch.cat(k.split(nq // G, dim=0), dim=1)
            v = torch.cat(v.split(nq // G, dim=0), dim=1)
        tgt2 = om.mha(sd, d + ".self_attn", q, k, v)
        tgt2 = torch.cat(tgt2.split(B, dim=1), dim=0).transpose(0, 1) if training else tgt2.transpose(0, 1)
        t = om.layer_norm(sd, d + ".norm2", t + om._drop(tgt2))
        tgt2 = om.ms_deform_attn(sd, d + ".cross_attn", t + query_pos, ref_in, memory, spatial_shapes)
        t = om.layer_norm(sd, d + ".norm1", t + om._drop(tgt2))
        output = om.layer_norm(sd, d + ".norm3", t + om._drop(om.linear(sd, d + ".linear2",
                                                                          om._drop(F.relu(om.linear(sd, d + ".linear1", t))))))
        tmp = om.mlp(sd, f"bbox_embed.{l}", output, 3)
        reference_points = (tmp + om.inverse_sigmoid(reference_points)).sigmoid().detach()
        inter.append(output)
        inter_ref.append(reference_points)
        inter_dim.append(om.mlp(sd, f"dim_embed_3d.{l}", output, 2))
    return torch.stack(inter), init_reference, torch.stack(inter_ref), torch.stack(inter_dim)


def deterministic_state_dict(cfg=CFG):
    """om.deterministic_state_dict's per-name weights over the use_dab names (shared names keep the default oracle's values).
    om draws each weight by name from the spec it looks up by module-global name, so that lookup is pointed at this module's
    spec for the duration of the call (the oracle package itself stays as it is)."""
    saved = om.state_dict_spec
    om.state_dict_spec = lambda c=cfg: state_dict_spec(c)
    try:
        return om.deterministic_state_dict(cfg)
    finally:
        om.state_dict_spec = saved


def forward(sd, images, calibs, img_sizes, training=False, cfg=CFG):
    """monodetr.py:150-283 with use_dab: om.forward's steps around this module's transformer.  The queries are
    cat(tgt_embed, refpoint_embed) rows as in monodetr.py:182-191."""
    feats = om.backbone(sd, images)
    B = images.shape[0]
    srcs = [om.conv_gn(sd, f"input_proj.{l}", f) for l, f in enumerate(feats)]
    srcs.append(om.conv_gn(sd, "input_proj.3", feats[-1], stride=2, padding=1))
    pos = [om.position_embedding_sine(B, s.shape[2], s.shape[3], s.device) for s in srcs]
    nq = cfg["num_queries"] * (cfg["group_num"] if training else 1)
    query_embeds = torch.cat((sd["tgt_embed.weight"], sd["refpoint_embed.weight"]), 1)[:nq]
    depth_logits, depth_pos_embed, weighted_depth, _ = om.depth_predictor(sd, srcs, pos[1], cfg)
    hs, init_ref, inter_refs, inter_dims = transformer(sd, srcs, pos, query_embeds, depth_pos_embed, training, cfg)
    coords, classes, dims, depths, angles = [], [], [], [], []
    for lvl in range(hs.shape[0]):
        coord = (om.mlp(sd, f"bbox_embed.{lvl}", hs[lvl], 3) + om.inverse_sigmoid(init_ref if lvl == 0 else inter_refs[lvl - 1])).sigmoid()
        coords.append(coord)
        classes.append(om.linear(sd, f"class_embed.{lvl}", hs[lvl]))
        size3d = inter_dims[lvl]
        dims.append(size3d)
        box_h = torch.clamp((coord[:, :, 4] + coord[:, :, 5]) * img_sizes[:, 1:2], min=1.0)
        depth_geo = size3d[:, :, 0] / box_h * calibs[:, 0, 0].unsqueeze(1)
        depth_reg = om.mlp(sd, f"depth_embed.{lvl}", hs[lvl], 2)
        centre = ((coord[..., :2] - 0.5) * 2).unsqueeze(2).detach()
        depth_map = F.grid_sample(weighted_depth.unsqueeze(1), centre, mode="bilinear", align_corners=True).squeeze(1)
        depths.append(torch.cat([((1. / (depth_reg[:, :, 0:1].sigmoid() + 1e-6) - 1.) + depth_geo.unsqueeze(-1) + depth_map) / 3,
                                 depth_reg[:, :, 1:2]], -1))
        angles.append(om.mlp(sd, f"angle_embed.{lvl}", hs[lvl], 2))
    out = {"pred_logits": classes[-1], "pred_boxes": coords[-1], "pred_3d_dim": dims[-1], "pred_depth": depths[-1],
           "pred_angle": angles[-1], "pred_depth_map_logits": depth_logits}
    out["aux_outputs"] = [{"pred_logits": a, "pred_boxes": b, "pred_3d_dim": c, "pred_angle": d, "pred_depth": e}
                          for a, b, c, d, e in zip(classes[:-1], coords[:-1], dims[:-1], angles[:-1], depths[:-1])]
    return out
