"""TEST INFRASTRUCTURE: the CPU oracle (oracle/monodetr_torch.py) for the reference's other head counts -- cfg["nheads"] 4 and
16 (head widths 64 and 16 at hidden_dim 256).  The reference's build_depthaware_transformer passes nheads to the encoder's and
the decoder's MSDeformAttn and to the decoder's two nn.MultiheadAttention (depth cross-attention, group self-attention); the
depth predictor's encoder keeps nhead=8 (depth_predictor.py:49).  oracle/monodetr_torch.py states the 8-head model; this
module restates only what the head count changes -- the mha / ms_deform_attn calls of the transformer, the MSDeformAttn
parameter shapes and the sampling-offset bias init -- and runs everything else through that module's own functions.  Pinned
to the unmodified reference by tests/test_nheads_host.py (tests/golden/nheads.npz)."""
import contextlib
import math

import torch

from oracle import monodetr_torch as om

_mha, _ms_deform_attn, _spec = om.mha, om.ms_deform_attn, om.state_dict_spec
TRANSFORMER = "depthaware_transformer."


def heads_cfg(nheads):
    """The oracle's cfg for a head count: om.CFG with nheads changed."""
    return dict(om.CFG, nheads=nheads)


def state_dict_spec(cfg):
    """om.state_dict_spec() with the MSDeformAttn projections sized for cfg["nheads"] (n_heads x 4 levels x 4 points)."""
    nh = cfg["nheads"]
    spec = dict(_spec(cfg))
    for name in spec:
        if ".sampling_offsets." in name:
            spec[name] = (nh * 4 * 4 * 2,) + spec[name][1:]
        elif ".attention_weights." in name:
            spec[name] = (nh * 4 * 4,) + spec[name][1:]
    return spec


@contextlib.contextmanager
def _variant(cfg):
    """om's model-level functions look mha / ms_deform_attn / the spec up by module-global name: point them at the head
    count's.  The depth predictor's encoder (prefix depth_predictor.) keeps 8 heads."""
    nh = cfg["nheads"]
    saved = om.mha, om.ms_deform_attn, om.state_dict_spec
    om.mha = lambda sd, p, q, k, v, nheads=8: _mha(sd, p, q, k, v, nh if p.startswith(TRANSFORMER) else nheads)
    om.ms_deform_attn = lambda sd, p, *a, n_heads=8, **kw: _ms_deform_attn(sd, p, *a, n_heads=nh, **kw)
    om.state_dict_spec = lambda c=cfg: state_dict_spec(c)
    try:
        yield
    finally:
        om.mha, om.ms_deform_attn, om.state_dict_spec = saved


def sampling_offsets_bias(nheads, n_levels=4, n_points=4):
    """ms_deform_attn.py:106-114: one unit direction per head, scaled by the point index + 1."""
    thetas = torch.arange(nheads, dtype=torch.float32) * (2.0 * math.pi / nheads)
    grid = torch.stack([thetas.cos(), thetas.sin()], -1)
    grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(nheads, 1, 1, 2).repeat(1, n_levels, n_points, 1)
    for i in range(n_points):
        grid[:, :, i, :] *= i + 1
    return grid.view(-1)


def deterministic_state_dict(cfg):
    """om.deterministic_state_dict's per-name weights over the head count's shapes, the sampling-offset biases laid out for
    cfg["nheads"] heads (at 8 heads every value equals om's)."""
    with _variant(cfg):
        sd = om.deterministic_state_dict(cfg)
    for name in sd:
        if name.endswith("sampling_offsets.bias"):
            sd[name] = sampling_offsets_bias(cfg["nheads"]).to(sd[name].dtype)
    return sd


def forward(sd, images, calibs, img_sizes, training=False, cfg=None):
    """om.forward with cfg["nheads"] heads in the transformer."""
    with _variant(cfg):
        return om.forward(sd, images, calibs, img_sizes, training=training, cfg=cfg)
