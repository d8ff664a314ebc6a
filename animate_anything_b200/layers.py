"""Parameter containers mirroring the `diffusers==0.24.0` leaf modules that the reference composes
(models/unet_3d_blocks.py:18-20, models/unet_3d_condition_mask.py:24-26).  Same attribute names, hence the same
`state_dict()` keys as the reference checkpoints (utils/convert_diffusers_to_original_ms_text_to_video.py:18-169).

These classes hold parameters only.  They deliberately have no torch `forward`: all arithmetic runs in the sm_90a
kernels driven by `engine.py`; calling them directly raises, so a silent eager fallback cannot happen.
"""
from __future__ import annotations

import torch
import torch.nn as nn


class _ParamsOnly(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError(f"{type(self).__name__} is a parameter container; the sm_90a engine executes it "
                           f"(animate_anything_b200.engine). There is no eager fallback.")


class TimestepEmbedding(_ParamsOnly):
    def __init__(self, in_channels, time_embed_dim, act_fn="silu", cond_proj_dim=None, out_dim=None):
        super().__init__()
        assert act_fn in ("silu", "swish")
        self.linear_1 = nn.Linear(in_channels, time_embed_dim)
        self.cond_proj = nn.Linear(cond_proj_dim, in_channels, bias=False) if cond_proj_dim is not None else None
        self.linear_2 = nn.Linear(time_embed_dim, out_dim if out_dim is not None else time_embed_dim)


class ResnetBlock2D(_ParamsOnly):
    def __init__(self, *, in_channels, out_channels=None, temb_channels=512, groups=32, eps=1e-6,
                 output_scale_factor=1.0, **unused):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.eps = eps
        self.groups = groups
        self.output_scale_factor = output_scale_factor
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps)
        self.conv1 = nn.Conv2d(in_channels, out_channels, 3, padding=1)
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(groups, out_channels, eps=eps)
        self.conv2 = nn.Conv2d(out_channels, out_channels, 3, padding=1)
        self.conv_shortcut = nn.Conv2d(in_channels, out_channels, 1) if in_channels != out_channels else None


class TemporalConvLayer(_ParamsOnly):
    def __init__(self, in_dim, out_dim=None, dropout=0.0):
        super().__init__()
        out_dim = out_dim or in_dim
        self.in_dim, self.out_dim = in_dim, out_dim
        self.conv1 = nn.Sequential(nn.GroupNorm(32, in_dim), nn.SiLU(),
                                   nn.Conv3d(in_dim, out_dim, (3, 1, 1), padding=(1, 0, 0)))
        self.conv2 = nn.Sequential(nn.GroupNorm(32, out_dim), nn.SiLU(), nn.Dropout(dropout),
                                   nn.Conv3d(out_dim, in_dim, (3, 1, 1), padding=(1, 0, 0)))
        self.conv3 = nn.Sequential(nn.GroupNorm(32, out_dim), nn.SiLU(), nn.Dropout(dropout),
                                   nn.Conv3d(out_dim, in_dim, (3, 1, 1), padding=(1, 0, 0)))
        self.conv4 = nn.Sequential(nn.GroupNorm(32, out_dim), nn.SiLU(), nn.Dropout(dropout),
                                   nn.Conv3d(out_dim, in_dim, (3, 1, 1), padding=(1, 0, 0)))
        nn.init.zeros_(self.conv4[-1].weight)
        nn.init.zeros_(self.conv4[-1].bias)


class Downsample2D(_ParamsOnly):
    def __init__(self, channels, use_conv=True, out_channels=None, padding=1, name="op"):
        super().__init__()
        assert use_conv
        self.channels, self.out_channels, self.padding = channels, out_channels or channels, padding
        self.conv = nn.Conv2d(channels, self.out_channels, 3, stride=2, padding=padding)


class Upsample2D(_ParamsOnly):
    def __init__(self, channels, use_conv=True, out_channels=None):
        super().__init__()
        assert use_conv
        self.channels, self.out_channels = channels, out_channels or channels
        self.conv = nn.Conv2d(channels, self.out_channels, 3, padding=1)


class Attention(_ParamsOnly):
    def __init__(self, query_dim, cross_attention_dim=None, heads=8, dim_head=64, bias=False, norm_num_groups=None,
                 eps=1e-5, residual_connection=False, rescale_output_factor=1.0):
        super().__init__()
        self.inner_dim = heads * dim_head
        self.heads, self.dim_head = heads, dim_head
        self.is_cross = cross_attention_dim is not None
        kv_dim = cross_attention_dim if cross_attention_dim is not None else query_dim
        self.residual_connection = residual_connection
        self.rescale_output_factor = rescale_output_factor
        self.group_norm = nn.GroupNorm(norm_num_groups, query_dim, eps=eps) if norm_num_groups is not None else None
        self.to_q = nn.Linear(query_dim, self.inner_dim, bias=bias)
        self.to_k = nn.Linear(kv_dim, self.inner_dim, bias=bias)
        self.to_v = nn.Linear(kv_dim, self.inner_dim, bias=bias)
        self.to_out = nn.ModuleList([nn.Linear(self.inner_dim, query_dim), nn.Dropout(0.0)])

    def set_processor(self, processor):   # surface used by train.py:132-135; the engine has one fused path
        pass


class GEGLU(_ParamsOnly):
    def __init__(self, dim_in, dim_out):
        super().__init__()
        self.proj = nn.Linear(dim_in, dim_out * 2)


class FeedForward(_ParamsOnly):
    def __init__(self, dim, mult=4):
        super().__init__()
        inner = dim * mult
        self.net = nn.ModuleList([GEGLU(dim, inner), nn.Dropout(0.0), nn.Linear(inner, dim)])


class BasicTransformerBlock(_ParamsOnly):
    def __init__(self, dim, num_attention_heads, attention_head_dim, cross_attention_dim=None,
                 double_self_attention=False, only_cross_attention=False):
        super().__init__()
        assert not only_cross_attention
        self.norm1 = nn.LayerNorm(dim)
        self.attn1 = Attention(dim, heads=num_attention_heads, dim_head=attention_head_dim)
        if cross_attention_dim is not None or double_self_attention:
            self.norm2 = nn.LayerNorm(dim)
            self.attn2 = Attention(dim, cross_attention_dim=None if double_self_attention else cross_attention_dim,
                                   heads=num_attention_heads, dim_head=attention_head_dim)
        else:
            self.norm2, self.attn2 = None, None
        self.norm3 = nn.LayerNorm(dim)
        self.ff = FeedForward(dim)


class Transformer2DModel(_ParamsOnly):
    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=None, num_layers=1,
                 norm_num_groups=32, cross_attention_dim=None, use_linear_projection=False,
                 only_cross_attention=False, upcast_attention=False):
        super().__init__()
        if not use_linear_projection:
            raise NotImplementedError("the reference builds Transformer2DModel with use_linear_projection=True "
                                      "(models/unet_3d_blocks.py:136,192)")
        inner = num_attention_heads * attention_head_dim
        self.heads, self.head_dim, self.in_channels = num_attention_heads, attention_head_dim, in_channels
        self.norm = nn.GroupNorm(norm_num_groups, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner, num_attention_heads, attention_head_dim,
                                  cross_attention_dim=cross_attention_dim) for _ in range(num_layers)])
        self.proj_out = nn.Linear(inner, in_channels)


class TransformerTemporalModel(_ParamsOnly):
    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=None, num_layers=1,
                 norm_num_groups=32, cross_attention_dim=None, double_self_attention=True):
        super().__init__()
        inner = num_attention_heads * attention_head_dim
        self.heads, self.head_dim, self.in_channels = num_attention_heads, attention_head_dim, in_channels
        self.norm = nn.GroupNorm(norm_num_groups, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner, num_attention_heads, attention_head_dim,
                                  cross_attention_dim=cross_attention_dim,
                                  double_self_attention=double_self_attention) for _ in range(num_layers)])
        self.proj_out = nn.Linear(inner, in_channels)
