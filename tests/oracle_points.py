"""TEST INFRASTRUCTURE: the CPU oracle (oracle/monodetr_torch.py) for the reference's other sampling-point counts --
cfg["enc_n_points"] / cfg["dec_n_points"], each any count from 1 to 8.  The reference's build_depthaware_transformer passes
enc_n_points to every encoder layer's MSDeformAttn and dec_n_points to every decoder layer's; the count sizes the
sampling_offsets / attention_weights projections, the sampling-offset bias init and the 6-d location scale (off / n_points).
oracle/monodetr_torch.py states the 4-point model; this module restates only what the counts change -- the ms_deform_attn calls
of the transformer, the MSDeformAttn parameter shapes and the sampling-offset bias init -- and runs everything else through that
module's own functions, so at 4 / 4 it equals the base oracle bit for bit.  Pinned to the unmodified reference by
tests/test_points_host.py (tests/golden/points.npz)."""
import contextlib
import math

import torch

from oracle import monodetr_torch as om

_ms_deform_attn, _spec = om.ms_deform_attn, om.state_dict_spec
ENCODER, DECODER = "depthaware_transformer.encoder.", "depthaware_transformer.decoder."


def points_cfg(enc, dec):
    """The oracle's cfg for a pair of point counts: om.CFG with enc_n_points / dec_n_points changed."""
    return dict(om.CFG, enc_n_points=enc, dec_n_points=dec)


def n_points_of(cfg, name):
    """The point count of the MSDeformAttn a parameter (or module prefix) belongs to, None outside the transformer's."""
    if name.startswith(ENCODER):
        return cfg["enc_n_points"]
    if name.startswith(DECODER):
        return cfg["dec_n_points"]
    return None


def state_dict_spec(cfg):
    """om.state_dict_spec() with each MSDeformAttn's projections sized for its point count (8 heads x 4 levels x P points)."""
    spec = dict(_spec(cfg))
    for name in spec:
        P = n_points_of(cfg, name)
        if ".sampling_offsets." in name:
            spec[name] = (8 * 4 * P * 2,) + spec[name][1:]
        elif ".attention_weights." in name and P is not None:
            spec[name] = (8 * 4 * P,) + spec[name][1:]
    return spec


@contextlib.contextmanager
def _variant(cfg):
    """om's model-level functions look ms_deform_attn / the spec up by module-global name: point them at the counts'."""
    saved = om.ms_deform_attn, om.state_dict_spec
    om.ms_deform_attn = lambda sd, p, *a, n_points=4, **kw: _ms_deform_attn(sd, p, *a, n_points=n_points_of(cfg, p), **kw)
    om.state_dict_spec = lambda c=cfg: state_dict_spec(c)
    try:
        yield
    finally:
        om.ms_deform_attn, om.state_dict_spec = saved


def sampling_offsets_bias(n_points, nheads=8, n_levels=4):
    """ms_deform_attn.py:106-114: one unit direction per head, scaled by the point index + 1."""
    thetas = torch.arange(nheads, dtype=torch.float32) * (2.0 * math.pi / nheads)
    grid = torch.stack([thetas.cos(), thetas.sin()], -1)
    grid = (grid / grid.abs().max(-1, keepdim=True)[0]).view(nheads, 1, 1, 2).repeat(1, n_levels, n_points, 1)
    for i in range(n_points):
        grid[:, :, i, :] *= i + 1
    return grid.view(-1)


def deterministic_state_dict(cfg):
    """om.deterministic_state_dict's per-name weights over the counts' shapes, the sampling-offset biases laid out for each
    layer's point count (at 4 / 4 every value equals om's)."""
    with _variant(cfg):
        sd = om.deterministic_state_dict(cfg)
    for name in sd:
        if name.endswith("sampling_offsets.bias"):
            sd[name] = sampling_offsets_bias(n_points_of(cfg, name)).to(sd[name].dtype)
    return sd


def forward(sd, images, calibs, img_sizes, training=False, cfg=None):
    """om.forward with cfg["enc_n_points"] / cfg["dec_n_points"] points in the transformer's deformable attention."""
    with _variant(cfg):
        return om.forward(sd, images, calibs, img_sizes, training=training, cfg=cfg)
