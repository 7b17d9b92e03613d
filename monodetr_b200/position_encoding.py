"""Position embeddings -- mirror of lib/models/monodetr/position_encoding.py for the all-False masks this path always has
(backbone.py:88, monodetr.py:173-174); layout is token-major (H*W, 256) to match NHWC activations.

  * PositionEmbeddingSine (:20-56, normalize=True, 128+128 features, temperature 10000): y_embed = (row+1)/(H+1e-6)*2pi, x_embed
    likewise, channels [pos_y | pos_x].  Input-independent, so it is computed once per (H, W, device) and cached.
  * PositionEmbeddingLearned (:59-86): two (50, 128) tables interpolated at x / W * 49 and y / H * 49, channels [col (x) | row (y)]
    -- the opposite order of the sine table.  Its tables train, so it is recomputed every call (one launch, csrc/pos_embed.cu).
"""
import math

import torch
from torch import nn

from . import functional as Fn


class PositionEmbeddingSine(nn.Module):
    def __init__(self, num_pos_feats=64, temperature=10000, normalize=False, scale=None):
        super().__init__()
        self.num_pos_feats = num_pos_feats
        self.temperature = temperature
        self.normalize = normalize
        if scale is not None and normalize is False:
            raise ValueError("normalize should be True if scale is passed")
        self.scale = 2 * math.pi if scale is None else scale
        self._cache = {}

    def table(self, H, W, device):
        key = (H, W, str(device))
        if key not in self._cache:
            y_embed = torch.arange(1, H + 1, dtype=torch.float32, device=device).view(H, 1).expand(H, W)
            x_embed = torch.arange(1, W + 1, dtype=torch.float32, device=device).view(1, W).expand(H, W)
            if self.normalize:
                eps = 1e-6
                y_embed = y_embed / (H + eps) * self.scale
                x_embed = x_embed / (W + eps) * self.scale
            dim_t = torch.arange(self.num_pos_feats, dtype=torch.float32, device=device)
            dim_t = self.temperature ** (2 * (dim_t // 2) / self.num_pos_feats)
            pos_x = x_embed[:, :, None] / dim_t
            pos_y = y_embed[:, :, None] / dim_t
            pos_x = torch.stack((pos_x[:, :, 0::2].sin(), pos_x[:, :, 1::2].cos()), dim=3).flatten(2)
            pos_y = torch.stack((pos_y[:, :, 0::2].sin(), pos_y[:, :, 1::2].cos()), dim=3).flatten(2)
            self._cache[key] = torch.cat((pos_y, pos_x), dim=2).reshape(H * W, -1).contiguous()
        return self._cache[key]

    def forward(self, feat_nhwc):
        """feat (B, H, W, C) -> (H*W, 2*num_pos_feats), identical for every image of the batch."""
        _, H, W, _ = feat_nhwc.shape
        return self.table(H, W, feat_nhwc.device)


class PositionEmbeddingLearned(nn.Module):
    """Same parameters (row_embed, col_embed: nn.Embedding(50, num_pos_feats), N(0, 1)) as the reference.  The kernels hold 128
    features per table (hidden_dim 256, which the depth predictor assumes as well)."""

    def __init__(self, num_pos_feats=256):
        super().__init__()
        if num_pos_feats != 128:
            raise NotImplementedError(f"monodetr_b200 position_embedding 'learned' implements hidden_dim 256 (num_pos_feats 128), "
                                      f"not num_pos_feats {num_pos_feats}")
        self.row_embed = nn.Embedding(50, num_pos_feats)
        self.col_embed = nn.Embedding(50, num_pos_feats)

    def forward(self, feat_nhwc):
        """feat (B, H, W, C) -> (H*W, 2*num_pos_feats) = [x_emb | y_emb], identical for every image of the batch."""
        _, H, W, _ = feat_nhwc.shape
        return Fn.pos_learned(self.col_embed.weight, self.row_embed.weight, H, W)


def build_position_encoding(cfg):
    n_steps = cfg["hidden_dim"] // 2
    if cfg["position_embedding"] in ("v2", "sine"):
        return PositionEmbeddingSine(n_steps, normalize=True)
    if cfg["position_embedding"] in ("v3", "learned"):
        return PositionEmbeddingLearned(n_steps)
    raise NotImplementedError("monodetr_b200 implements position_embedding: 'sine' / 'v2' and 'learned' / 'v3' "
                              "(configs/monodetr.yaml)")
