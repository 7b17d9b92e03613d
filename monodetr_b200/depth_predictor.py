"""Foreground-depth predictor -- mirror of lib/models/monodetr/depth_predictor/depth_predictor.py:7-104 and
depth_predictor/transformer.py:16-65 (same parameter names) on the sm_90a kernels.  Activations are NHWC /
token-major; convs are the wgmma implicit-GEMM kernel, GroupNorm(+ReLU), attention and LayerNorm are the fused
kernels of csrc/norm.cu / attention.cu."""
import copy

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib, functional as Fn


class TransformerEncoderLayer(nn.Module):
    def __init__(self, d_model, nhead, dim_feedforward=2048, dropout=0.1, site_base=900):
        super().__init__()
        self.self_attn = nn.MultiheadAttention(d_model, nhead, dropout=dropout)      # parameter container
        self.linear1 = nn.Linear(d_model, dim_feedforward)
        self.dropout = nn.Dropout(dropout)
        self.linear2 = nn.Linear(dim_feedforward, d_model)
        self.norm1 = nn.LayerNorm(d_model)
        self.norm2 = nn.LayerNorm(d_model)
        self.dropout1 = nn.Dropout(dropout)
        self.dropout2 = nn.Dropout(dropout)
        self.site_base = site_base

    def forward(self, src, src_key_padding_mask, pos):
        """src (B, L, C) batch-first, pos (L, C) or (B, L, C)."""
        a = self.self_attn
        c = src.shape[-1]
        qk_in = src + pos
        qk = Fn.linear(qk_in, a.in_proj_weight[:2 * c], a.in_proj_bias[:2 * c])            # fused q,k projection
        v = Fn.linear(src, a.in_proj_weight[2 * c:], a.in_proj_bias[2 * c:])
        o = Fn.attention(qk[..., :c], qk[..., c:], v, src_key_padding_mask, a.dropout, self.training, self.site_base)
        src2 = Fn.linear(o, a.out_proj.weight, a.out_proj.bias)
        src = Fn.add_layernorm(src, src2, self.norm1.weight, self.norm1.bias, self.norm1.eps, self.dropout1.p,
                               self.training, self.site_base + 1)
        h = Fn.linear(src, self.linear1.weight, self.linear1.bias, relu=True)
        h = Fn.dropout(h, self.dropout.p, self.training, self.site_base + 2)
        src2 = Fn.linear(h, self.linear2.weight, self.linear2.bias)
        return Fn.add_layernorm(src, src2, self.norm2.weight, self.norm2.bias, self.norm2.eps, self.dropout2.p,
                                self.training, self.site_base + 3)


class TransformerEncoder(nn.Module):
    def __init__(self, encoder_layer, num_layers, norm=None):
        super().__init__()
        self.layers = nn.ModuleList([copy.deepcopy(encoder_layer) for _ in range(num_layers)])
        self.num_layers = num_layers
        self.norm = norm

    def forward(self, src, src_key_padding_mask, pos):
        for layer in self.layers:
            src = layer(src, src_key_padding_mask, pos)
        return src


class _ConvGN(nn.Sequential):
    """Sequential(Conv2d, GroupNorm(32, C)) parameter container with an NHWC forward."""

    def __init__(self, cin, cout, k, stride=1, padding=0):
        super().__init__(nn.Conv2d(cin, cout, kernel_size=k, stride=stride, padding=padding), nn.GroupNorm(32, cout))

    def forward(self, x, relu=False):
        conv, gn = self[0], self[1]
        y = Fn.conv2d_nhwc(x, conv.weight, conv.bias, conv.stride[0], conv.padding[0])
        return Fn.groupnorm_nhwc(y, gn.weight, gn.bias, gn.num_groups, gn.eps, relu)


def library_resize(x):
    """Whether the 1/32 map is resized with the library's kernel (mdb_upsample_bilinear_nhwc_*) instead of F.interpolate: in
    reproducible mode, for a map on a CUDA device, because torch's CUDA backward of the bilinear resize scatters with atomics
    (and raises under torch.use_deterministic_algorithms(True)).  Its CPU backward -- reached only by the host-logic tests,
    which drive the model with CPU tensors -- is deterministic, and the default mode keeps F.interpolate everywhere."""
    return _lib.deterministic() and x.device.type == "cuda"


class DepthPredictor(nn.Module):
    def __init__(self, model_cfg):
        super().__init__()
        depth_num_bins = int(model_cfg["num_depth_bins"])
        depth_min = float(model_cfg["depth_min"])
        depth_max = float(model_cfg["depth_max"])
        self.depth_max = depth_max
        bin_size = 2 * (depth_max - depth_min) / (depth_num_bins * (1 + depth_num_bins))
        bin_indice = torch.linspace(0, depth_num_bins - 1, depth_num_bins)
        bin_value = (bin_indice + 0.5).pow(2) * bin_size / 2 - bin_size / 8 + depth_min
        bin_value = torch.cat([bin_value, torch.tensor([depth_max])], dim=0)
        self.depth_bin_values = nn.Parameter(bin_value, requires_grad=False)
        d_model = model_cfg["hidden_dim"]
        self.downsample = _ConvGN(d_model, d_model, 3, 2, 1)
        self.proj = _ConvGN(d_model, d_model, 1)
        self.upsample = _ConvGN(d_model, d_model, 1)
        self.depth_head = nn.Sequential(
            nn.Conv2d(d_model, d_model, kernel_size=(3, 3), padding=1), nn.GroupNorm(32, num_channels=d_model), nn.ReLU(),
            nn.Conv2d(d_model, d_model, kernel_size=(3, 3), padding=1), nn.GroupNorm(32, num_channels=d_model), nn.ReLU())
        self.depth_classifier = nn.Conv2d(d_model, depth_num_bins + 1, kernel_size=(1, 1))
        self.depth_encoder = TransformerEncoder(TransformerEncoderLayer(d_model, nhead=8, dim_feedforward=256, dropout=0.1), 1)
        self.depth_pos_embed = nn.Embedding(int(self.depth_max) + 1, 256)

    def forward(self, feature, mask, pos):
        """feature: 4 NHWC maps (B, H_l, W_l, C); mask (B, H1*W1) bool or None; pos (H1*W1, C).
        Returns depth_logits (B, H, W, 81) NHWC, depth_embed (B, HW, C), weighted_depth (B, H, W),
        depth_pos_embed_ip (B, HW, C)  -- the reference's (:91) tensors in channels-last layout."""
        assert len(feature) == 4
        src_16 = self.proj(feature[1])
        if library_resize(feature[2]):
            up = Fn.upsample_bilinear_nhwc(feature[2], src_16.shape[1:3])
        else:
            up = F.interpolate(feature[2].permute(0, 3, 1, 2), size=src_16.shape[1:3], mode="bilinear").permute(0, 2, 3, 1)
        src_32 = self.upsample(up.contiguous())
        src_8 = self.downsample(feature[0])
        src = Fn.mean3(src_8, src_16, src_32)
        h = self.depth_head
        src = Fn.groupnorm_nhwc(Fn.conv2d_nhwc(src, h[0].weight, h[0].bias, 1, 1), h[1].weight, h[1].bias, 32, h[1].eps, True)
        src = Fn.groupnorm_nhwc(Fn.conv2d_nhwc(src, h[3].weight, h[3].bias, 1, 1), h[4].weight, h[4].bias, 32, h[4].eps, True)
        depth_logits = Fn.conv2d_nhwc(src, self.depth_classifier.weight, self.depth_classifier.bias, 1, 0)
        # softmax over the bins -> expected depth -> lerp into the depth positional embedding (:74-77, :93-104), one kernel
        weighted_depth, depth_pos_embed_ip = Fn.depth_tail(depth_logits, self.depth_bin_values, self.depth_pos_embed.weight, self.depth_max)
        B, H, W, C = src.shape
        depth_embed = self.depth_encoder(src.view(B, H * W, C), mask, pos)
        depth_pos_embed_ip = depth_pos_embed_ip.view(B, H * W, C)
        return depth_logits, depth_embed + depth_pos_embed_ip, weighted_depth, depth_pos_embed_ip

    def interpolate_depth_embed(self, depth):
        depth = depth.clamp(min=0, max=self.depth_max)
        return self.interpolate_1d(depth, self.depth_pos_embed)

    def interpolate_1d(self, coord, embed):
        floor_coord = coord.floor()
        delta = (coord - floor_coord).unsqueeze(-1)
        floor_coord = floor_coord.long()
        ceil_coord = (floor_coord + 1).clamp(max=embed.num_embeddings - 1)
        return embed(floor_coord) * (1 - delta) + embed(ceil_coord) * delta
