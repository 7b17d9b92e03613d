"""MSDeformAttn module -- mirror of lib/models/monodetr/ops/modules/ms_deform_attn.py:69-162 (same parameters,
same initialisation :106-120, same forward contract) on the sm_90a kernels: the four projections are tensor-core
GEMMs, the sampling core is csrc/msda.cu.  Batch-first tensors (N, Len, C) as in the reference."""
import math

import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.init import constant_, xavier_uniform_

from . import functional as Fn


class MSDeformAttn(nn.Module):
    # Test switch (default off): treat the sampling locations as constants in backward.  d(bilinear)/d(location) is
    # discontinuous at cell borders; with it frozen every remaining gradient of the model is smooth and can be held to a
    # tight tolerance against the CPU oracle (tests/test_model_grad_gpu.py).
    freeze_sampling_locations = False

    def __init__(self, d_model=256, n_levels=4, n_heads=8, n_points=4):
        super().__init__()
        if d_model % n_heads != 0:
            raise ValueError(f"d_model must be divisible by n_heads, but got {d_model} and {n_heads}")
        self.im2col_step = 64
        self.d_model, self.n_levels, self.n_heads, self.n_points = d_model, n_levels, n_heads, n_points
        self.sampling_offsets = nn.Linear(d_model, n_heads * n_levels * n_points * 2)
        self.attention_weights = nn.Linear(d_model, n_heads * n_levels * n_points)
        self.value_proj = nn.Linear(d_model, d_model)
        self.output_proj = nn.Linear(d_model, d_model)
        self._reset_parameters()

    def _reset_parameters(self):
        constant_(self.sampling_offsets.weight.data, 0.)
        thetas = torch.arange(self.n_heads, dtype=torch.float32) * (2.0 * math.pi / self.n_heads)
        grid_init = torch.stack([thetas.cos(), thetas.sin()], -1)
        grid_init = (grid_init / grid_init.abs().max(-1, keepdim=True)[0]).view(self.n_heads, 1, 1, 2) \
            .repeat(1, self.n_levels, self.n_points, 1)
        for i in range(self.n_points):
            grid_init[:, :, i, :] *= i + 1
        with torch.no_grad():
            self.sampling_offsets.bias = nn.Parameter(grid_init.view(-1))
        constant_(self.attention_weights.weight.data, 0.)
        constant_(self.attention_weights.bias.data, 0.)
        xavier_uniform_(self.value_proj.weight.data)
        constant_(self.value_proj.bias.data, 0.)
        xavier_uniform_(self.output_proj.weight.data)
        constant_(self.output_proj.bias.data, 0.)

    def project_value(self, input_flatten, input_padding_mask=None):
        """value_proj + padding fill (:136-139): depends on the memory only, so a caller may run it ahead of the query path."""
        N, Len_in, _ = input_flatten.shape
        value = Fn.linear(input_flatten, self.value_proj.weight, self.value_proj.bias)
        if input_padding_mask is not None:
            value = value.masked_fill(input_padding_mask[..., None], float(0))
        return value.view(N, Len_in, self.n_heads, self.d_model // self.n_heads)

    def forward(self, query, reference_points, input_flatten, input_spatial_shapes, input_level_start_index,
                input_padding_mask=None, value=None):
        """Same arguments as the reference (:122-134) (+ `value`: the result of `project_value`, if already computed);
        returns (N, Len_q, C)."""
        N, Len_q, _ = query.shape
        if value is None:
            value = self.project_value(input_flatten, input_padding_mask)
        sampling_offsets = Fn.linear(query, self.sampling_offsets.weight, self.sampling_offsets.bias)
        attention_logits = Fn.linear(query, self.attention_weights.weight, self.attention_weights.bias)
        if self.freeze_sampling_locations:
            sampling_offsets, reference_points = sampling_offsets.detach(), reference_points.detach()
        if reference_points.shape[-1] not in (2, 6):
            raise ValueError(f"Last dim of reference_points must be 2 or 6, but get {reference_points.shape[-1]} instead.")
        if reference_points.dim() == 2:
            # (Len_q, 6) boxes shared by every image and level (use_dab's anchors at decoder layer 0): differentiable in the boxes
            if reference_points.shape[-1] != 6:
                raise ValueError("shared reference boxes must be (Len_q, 6)")
            output = Fn.msda_shared_boxes(value, input_spatial_shapes, input_level_start_index, sampling_offsets, attention_logits,
                                          reference_points, self.n_heads, self.n_levels, self.n_points)
            return Fn.linear(output, self.output_proj.weight, self.output_proj.bias)
        # :145-155 fused: softmax over the L*P (level, point) logits and loc = ref + off / (W_l, H_l)   [2-d refs]
        #                                                     or ref_xy + off / P * (l+r, t+b) / 2    [6-d refs]
        if Fn.msda_fused_applicable(value, reference_points, self.n_levels, self.n_points):
            # constant reference points (the encoder's pixel grid; decoder layers 1-2, whose boxes are detached): the
            # pre-processing runs inside the sampling kernels
            output = Fn.msda_fused(value, input_spatial_shapes, input_level_start_index, sampling_offsets, attention_logits,
                                   reference_points)
        else:
            sampling_locations, attention_weights = Fn.msda_prep(sampling_offsets, attention_logits, reference_points,
                                                                input_spatial_shapes, self.n_heads, self.n_levels, self.n_points)
            output = Fn.msda(value, input_spatial_shapes, input_level_start_index, sampling_locations, attention_weights)
        return Fn.linear(output, self.output_proj.weight, self.output_proj.bias)
