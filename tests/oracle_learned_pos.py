"""TEST INFRASTRUCTURE: the CPU oracle (oracle/monodetr_torch.py) for the learned position embedding (`position_embedding:
'learned'`).

oracle/monodetr_torch.py states the sine embedding; this module restates PositionEmbeddingLearned (position_encoding.py:59-86) --
two (50, 128) tables `backbone.1.row_embed.weight` / `backbone.1.col_embed.weight`, interpolated at x / w * 49, channels
[col (x) | row (y)] -- and runs every model-level function of that module (or of tests/oracle_dab.py / tests/oracle_backbones.py,
which call it) with it in place of the sine embedding.  Pinned to the unmodified reference by tests/test_oracle_learned_pos.py
(tests/golden/learned_pos.npz)."""
import contextlib
import hashlib

import numpy as np
import torch

from oracle import monodetr_torch as om

ROW, COL = "backbone.1.row_embed.weight", "backbone.1.col_embed.weight"
TABLE_SHAPE = (50, 128)
# the module-alone shapes of the fixture: w = 49 (integer coordinates), w > 50, h > 50, w = 1 and the model's level shapes
SHAPES = ((1, 1), (1, 49), (2, 50), (3, 51), (7, 333), (60, 7), (48, 160), (24, 80), (12, 40), (6, 20))
MODULE_SEED = 7
GRAD_SAMPLES = 256


def module_tables():
    """(col, row): the seeded (50, 128) tables of the module-alone check, N(0, 1), col drawn first."""
    g = torch.Generator().manual_seed(MODULE_SEED)
    col = torch.randn(TABLE_SHAPE, generator=g)
    return col, torch.randn(TABLE_SHAPE, generator=g)


def upstream_grad(h, w):
    """The seeded upstream gradient of the module-alone check, in the reference's (1, 256, h, w) layout."""
    return torch.randn((1, 256, h, w), generator=torch.Generator().manual_seed(1000 * h + w))


def digest(t):
    """SHA-256 of a float32 tensor's values in row-major order, as a uint8 array: a bit-exact check that stores 32 bytes."""
    a = np.ascontiguousarray(t.detach().cpu().numpy().astype(np.float32, copy=False))
    return np.frombuffer(hashlib.sha256(a.tobytes()).digest(), dtype=np.uint8)


def grad_sample_index(g, key):
    """GRAD_SAMPLES flat positions of a table gradient, drawn (seeded by `key`) among its non-zero entries (all of them if fewer):
    the rows a small map never reaches are zero and would say nothing."""
    nz = np.flatnonzero(g.detach().cpu().numpy().reshape(-1))
    if nz.size <= GRAD_SAMPLES:
        return nz.astype(np.int32)
    rng = np.random.default_rng(sum(key.encode()))
    return np.sort(rng.choice(nz, GRAD_SAMPLES, replace=False)).astype(np.int32)


def get_embed(coord, table):
    """position_encoding.py:81-86: table rows floor(coord) and min(floor + 1, 49), blended by the fraction."""
    floor_coord = coord.floor()
    delta = (coord - floor_coord).unsqueeze(-1)
    floor_coord = floor_coord.long()
    ceil_coord = (floor_coord + 1).clamp(max=table.shape[0] - 1)
    return table[floor_coord] * (1 - delta) + table[ceil_coord] * delta


def axis_embeds(col, row, H, W):
    """(x_emb (W, 128), y_emb (H, 128)) as position_encoding.py:68-74 computes them."""
    i = torch.arange(W, device=col.device) / W * 49
    j = torch.arange(H, device=row.device) / H * 49
    return get_embed(i, col), get_embed(j, row)


def position_embedding_learned(col, row, B, H, W):
    """position_encoding.py:68-79 for a (B, C, H, W) map: (B, 256, H, W), identical for every image."""
    x_emb, y_emb = axis_embeds(col, row, H, W)
    pos = torch.cat([x_emb.unsqueeze(0).expand(H, -1, -1), y_emb.unsqueeze(1).expand(-1, W, -1)], dim=-1).permute(2, 0, 1)
    return pos.unsqueeze(0).expand(B, -1, -1, -1)


def table_nhwc(col, row, H, W):
    """The product's layout of the same table: (H*W, 256), token-major."""
    return position_embedding_learned(col, row, 1, H, W)[0].permute(1, 2, 0).reshape(H * W, -1)


def state_dict_spec(base_spec):
    """A spec (name -> shape, om.state_dict_spec or a variant's) with the two tables."""
    return dict(base_spec, **{ROW: TABLE_SHAPE, COL: TABLE_SHAPE})


def with_tables(sd):
    """A deterministic state dict (om.deterministic_state_dict or a variant's) plus the two tables, drawn by name with om's rule
    for embedding weights (N(0, 1) from the name's seed)."""
    out = dict(sd)
    for name in (ROW, COL):
        out[name] = torch.randn(TABLE_SHAPE, generator=torch.Generator().manual_seed(om._seed_of(name)))
    return out


@contextlib.contextmanager
def learned(sd):
    """om's model-level functions look the position embedding up by module-global name: point it at sd's learned tables."""
    saved = om.position_embedding_sine
    om.position_embedding_sine = lambda B, H, W, device, *a: position_embedding_learned(sd[COL], sd[ROW], B, H, W)
    try:
        yield
    finally:
        om.position_embedding_sine = saved


def forward(sd, images, calibs, img_sizes, training=False, base=om.forward, **kw):
    """`base` (om.forward, oracle_dab.forward, oracle_backbones.forward, ...) with the learned embedding."""
    with learned(sd):
        return base(sd, images, calibs, img_sizes, training=training, **kw)
