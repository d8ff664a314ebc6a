"""Mirror of the reference's `models/unet_3d_blocks.py` block classes: same class names, constructor arguments,
sub-module attribute names (-> identical state_dict keys) and layer order, executed on the sm_90a engine.

Layer order per the reference:
  CrossAttnDownBlock3D / CrossAttnUpBlock3D: resnet -> temp_conv -> attn -> temp_attn   (unet_3d_blocks.py:514-526,747-759)
  UNetMidBlock3DCrossAttn: resnet0, temp_conv0, then (attn, temp_attn, resnet, temp_conv)               (:353-384)
  DownBlock3D / UpBlock3D: resnet -> temp_conv                                                         (:606-609,833-836)
Temporal modules are skipped when num_frames == 1 (:516,525,378,383).  The gradient-checkpoint wrappers (:32-120) are
training-only and out of scope.
"""
from __future__ import annotations

import torch.nn as nn

from . import engine as E
from .layers import (Downsample2D, ResnetBlock2D, TemporalConvLayer, Transformer2DModel, TransformerTemporalModel,
                     Upsample2D)


def _resnet(cin, cout, temb, eps, groups, scale=1.0):
    return ResnetBlock2D(in_channels=cin, out_channels=cout, temb_channels=temb, eps=eps, groups=groups,
                         output_scale_factor=scale)


def _spatial(c, head_ch, cross_dim, groups, use_linear_projection):
    return Transformer2DModel(c // head_ch, head_ch, in_channels=c, num_layers=1, cross_attention_dim=cross_dim,
                              norm_num_groups=groups, use_linear_projection=use_linear_projection)


def _temporal(c, head_ch, cross_dim, groups):
    return TransformerTemporalModel(c // head_ch, head_ch, in_channels=c, num_layers=1, cross_attention_dim=cross_dim,
                                    norm_num_groups=groups)


class _Block(nn.Module):
    gradient_checkpointing = False

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("blocks are executed through UNet3DConditionModel.forward (sm_90a engine)")


class UNetMidBlock3DCrossAttn(_Block):
    def __init__(self, in_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 attn_num_head_channels=1, output_scale_factor=1.0, cross_attention_dim=1280,
                 dual_cross_attention=False, use_linear_projection=True, upcast_attention=False):
        super().__init__()
        self.has_cross_attention = True
        self.attn_num_head_channels = attn_num_head_channels
        resnet_groups = resnet_groups if resnet_groups is not None else min(in_channels // 4, 32)
        resnets = [_resnet(in_channels, in_channels, temb_channels, resnet_eps, resnet_groups, output_scale_factor)]
        temp_convs = [TemporalConvLayer(in_channels, in_channels, dropout=0.1)]
        attentions, temp_attentions = [], []
        for _ in range(num_layers):
            attentions.append(_spatial(in_channels, attn_num_head_channels, cross_attention_dim, resnet_groups,
                                       use_linear_projection))
            temp_attentions.append(_temporal(in_channels, attn_num_head_channels, cross_attention_dim, resnet_groups))
            resnets.append(_resnet(in_channels, in_channels, temb_channels, resnet_eps, resnet_groups,
                                   output_scale_factor))
            temp_convs.append(TemporalConvLayer(in_channels, in_channels, dropout=0.1))
        self.resnets = nn.ModuleList(resnets)
        self.temp_convs = nn.ModuleList(temp_convs)
        self.attentions = nn.ModuleList(attentions)
        self.temp_attentions = nn.ModuleList(temp_attentions)

    def run(self, ctx, x, g):
        x = E.resnet_forward(ctx, self.resnets[0], x, g)
        x = E.temporal_conv_forward(ctx, self.temp_convs[0], x, g)   # reference :354 (no num_frames guard)
        for attn, tattn, resnet, tconv in zip(self.attentions, self.temp_attentions, self.resnets[1:],
                                              self.temp_convs[1:]):
            x, g = E.spatial_transformer_forward(ctx, attn, x, g)
            if g.t > 1:
                x = E.temporal_transformer_forward(ctx, tattn, x, g)
            x = E.resnet_forward(ctx, resnet, x, g)
            if g.t > 1:
                x = E.temporal_conv_forward(ctx, tconv, x, g)
        return x, g      # g changes when the shared CFG prefix ends inside this block (all-DownBlock3D configs)


class CrossAttnDownBlock3D(_Block):
    def __init__(self, in_channels, out_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 attn_num_head_channels=1, cross_attention_dim=1280, output_scale_factor=1.0, downsample_padding=1,
                 add_downsample=True, dual_cross_attention=False, use_linear_projection=False,
                 only_cross_attention=False, upcast_attention=False):
        super().__init__()
        self.has_cross_attention = True
        self.attn_num_head_channels = attn_num_head_channels
        resnets, temp_convs, attentions, temp_attentions = [], [], [], []
        for i in range(num_layers):
            cin = in_channels if i == 0 else out_channels
            resnets.append(_resnet(cin, out_channels, temb_channels, resnet_eps, resnet_groups, output_scale_factor))
            temp_convs.append(TemporalConvLayer(out_channels, out_channels, dropout=0.1))
            attentions.append(_spatial(out_channels, attn_num_head_channels, cross_attention_dim, resnet_groups,
                                       use_linear_projection))
            temp_attentions.append(_temporal(out_channels, attn_num_head_channels, cross_attention_dim, resnet_groups))
        self.resnets = nn.ModuleList(resnets)
        self.temp_convs = nn.ModuleList(temp_convs)
        self.attentions = nn.ModuleList(attentions)
        self.temp_attentions = nn.ModuleList(temp_attentions)
        self.downsamplers = (nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                         padding=downsample_padding, name="op")])
                             if add_downsample else None)

    def run(self, ctx, x, g):
        outs = []
        for resnet, tconv, attn, tattn in zip(self.resnets, self.temp_convs, self.attentions, self.temp_attentions):
            x = E.resnet_forward(ctx, resnet, x, g)
            if g.t > 1:
                x = E.temporal_conv_forward(ctx, tconv, x, g)
            x, g = E.spatial_transformer_forward(ctx, attn, x, g)
            if g.t > 1:
                x = E.temporal_transformer_forward(ctx, tattn, x, g)
            outs.append((x, g))
        if self.downsamplers is not None:
            x = E.downsample_forward(ctx, self.downsamplers[0], x, g)
            g = g.down()
            outs.append((x, g))
        return x, g, outs


class DownBlock3D(_Block):
    def __init__(self, in_channels, out_channels, temb_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True,
                 output_scale_factor=1.0, add_downsample=True, downsample_padding=1):
        super().__init__()
        resnets, temp_convs = [], []
        for i in range(num_layers):
            cin = in_channels if i == 0 else out_channels
            resnets.append(_resnet(cin, out_channels, temb_channels, resnet_eps, resnet_groups, output_scale_factor))
            temp_convs.append(TemporalConvLayer(out_channels, out_channels, dropout=0.1))
        self.resnets = nn.ModuleList(resnets)
        self.temp_convs = nn.ModuleList(temp_convs)
        self.downsamplers = (nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                         padding=downsample_padding, name="op")])
                             if add_downsample else None)

    def run(self, ctx, x, g):
        outs = []
        for resnet, tconv in zip(self.resnets, self.temp_convs):
            x = E.resnet_forward(ctx, resnet, x, g)
            if g.t > 1:
                x = E.temporal_conv_forward(ctx, tconv, x, g)
            outs.append((x, g))
        if self.downsamplers is not None:
            x = E.downsample_forward(ctx, self.downsamplers[0], x, g)
            g = g.down()
            outs.append((x, g))
        return x, g, outs


class CrossAttnUpBlock3D(_Block):
    def __init__(self, in_channels, out_channels, prev_output_channel, temb_channels, dropout=0.0, num_layers=1,
                 resnet_eps=1e-6, resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32,
                 resnet_pre_norm=True, attn_num_head_channels=1, cross_attention_dim=1280, output_scale_factor=1.0,
                 add_upsample=True, dual_cross_attention=False, use_linear_projection=False,
                 only_cross_attention=False, upcast_attention=False):
        super().__init__()
        self.has_cross_attention = True
        self.attn_num_head_channels = attn_num_head_channels
        resnets, temp_convs, attentions, temp_attentions = [], [], [], []
        for i in range(num_layers):
            skip_ch = in_channels if (i == num_layers - 1) else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(_resnet(cin + skip_ch, out_channels, temb_channels, resnet_eps, resnet_groups,
                                   output_scale_factor))
            temp_convs.append(TemporalConvLayer(out_channels, out_channels, dropout=0.1))
            attentions.append(_spatial(out_channels, attn_num_head_channels, cross_attention_dim, resnet_groups,
                                       use_linear_projection))
            temp_attentions.append(_temporal(out_channels, attn_num_head_channels, cross_attention_dim, resnet_groups))
        self.resnets = nn.ModuleList(resnets)
        self.temp_convs = nn.ModuleList(temp_convs)
        self.attentions = nn.ModuleList(attentions)
        self.temp_attentions = nn.ModuleList(temp_attentions)
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)

    def run(self, ctx, x, g, skips, upsample_size=None):
        for resnet, tconv, attn, tattn in zip(self.resnets, self.temp_convs, self.attentions, self.temp_attentions):
            skip, sg = skips.pop()
            assert (sg.h, sg.w) == (g.h, g.w)
            if sg.b * 2 == g.b:                       # skip produced inside the shared CFG prefix (batch b/2)
                skip = E.ops.dup_rows(skip)
            x = E.resnet_forward(ctx, resnet, x, g, skip=skip)
            if g.t > 1:
                x = E.temporal_conv_forward(ctx, tconv, x, g)
            x, g = E.spatial_transformer_forward(ctx, attn, x, g)
            if g.t > 1:
                x = E.temporal_transformer_forward(ctx, tattn, x, g)
        if self.upsamplers is not None:
            x = E.upsample_forward(ctx, self.upsamplers[0], x, g, size=upsample_size)
            g = g.up() if upsample_size is None else E.Geo(g.b, g.t, upsample_size[0], upsample_size[1])
        return x, g


class UpBlock3D(_Block):
    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, dropout=0.0, num_layers=1,
                 resnet_eps=1e-6, resnet_time_scale_shift="default", resnet_act_fn="swish", resnet_groups=32,
                 resnet_pre_norm=True, output_scale_factor=1.0, add_upsample=True):
        super().__init__()
        resnets, temp_convs = [], []
        for i in range(num_layers):
            skip_ch = in_channels if (i == num_layers - 1) else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(_resnet(cin + skip_ch, out_channels, temb_channels, resnet_eps, resnet_groups,
                                   output_scale_factor))
            temp_convs.append(TemporalConvLayer(out_channels, out_channels, dropout=0.1))
        self.resnets = nn.ModuleList(resnets)
        self.temp_convs = nn.ModuleList(temp_convs)
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)

    def run(self, ctx, x, g, skips, upsample_size=None):
        for resnet, tconv in zip(self.resnets, self.temp_convs):
            skip, sg = skips.pop()
            assert (sg.h, sg.w) == (g.h, g.w)
            if sg.b * 2 == g.b:                       # skip produced inside the shared CFG prefix (batch b/2)
                skip = E.ops.dup_rows(skip)
            x = E.resnet_forward(ctx, resnet, x, g, skip=skip)
            if g.t > 1:
                x = E.temporal_conv_forward(ctx, tconv, x, g)
        if self.upsamplers is not None:
            x = E.upsample_forward(ctx, self.upsamplers[0], x, g, size=upsample_size)
            g = g.up() if upsample_size is None else E.Geo(g.b, g.t, upsample_size[0], upsample_size[1])
        return x, g


def get_down_block(down_block_type, num_layers, in_channels, out_channels, temb_channels, add_downsample, resnet_eps,
                   resnet_act_fn, attn_num_head_channels, resnet_groups=None, cross_attention_dim=None,
                   downsample_padding=None, dual_cross_attention=False, use_linear_projection=True,
                   only_cross_attention=False, upcast_attention=False, resnet_time_scale_shift="default"):
    if down_block_type == "DownBlock3D":
        return DownBlock3D(num_layers=num_layers, in_channels=in_channels, out_channels=out_channels,
                           temb_channels=temb_channels, add_downsample=add_downsample, resnet_eps=resnet_eps,
                           resnet_act_fn=resnet_act_fn, resnet_groups=resnet_groups,
                           downsample_padding=downsample_padding)
    if down_block_type == "CrossAttnDownBlock3D":
        if cross_attention_dim is None:
            raise ValueError("cross_attention_dim must be specified for CrossAttnDownBlock3D")
        return CrossAttnDownBlock3D(num_layers=num_layers, in_channels=in_channels, out_channels=out_channels,
                                    temb_channels=temb_channels, add_downsample=add_downsample, resnet_eps=resnet_eps,
                                    resnet_act_fn=resnet_act_fn, resnet_groups=resnet_groups,
                                    downsample_padding=downsample_padding, cross_attention_dim=cross_attention_dim,
                                    attn_num_head_channels=attn_num_head_channels,
                                    use_linear_projection=use_linear_projection)
    raise ValueError(f"{down_block_type} does not exist.")


def get_up_block(up_block_type, num_layers, in_channels, out_channels, prev_output_channel, temb_channels,
                 add_upsample, resnet_eps, resnet_act_fn, attn_num_head_channels, resnet_groups=None,
                 cross_attention_dim=None, dual_cross_attention=False, use_linear_projection=True,
                 only_cross_attention=False, upcast_attention=False, resnet_time_scale_shift="default"):
    if up_block_type == "UpBlock3D":
        return UpBlock3D(num_layers=num_layers, in_channels=in_channels, out_channels=out_channels,
                         prev_output_channel=prev_output_channel, temb_channels=temb_channels,
                         add_upsample=add_upsample, resnet_eps=resnet_eps, resnet_act_fn=resnet_act_fn,
                         resnet_groups=resnet_groups)
    if up_block_type == "CrossAttnUpBlock3D":
        if cross_attention_dim is None:
            raise ValueError("cross_attention_dim must be specified for CrossAttnUpBlock3D")
        return CrossAttnUpBlock3D(num_layers=num_layers, in_channels=in_channels, out_channels=out_channels,
                                  prev_output_channel=prev_output_channel, temb_channels=temb_channels,
                                  add_upsample=add_upsample, resnet_eps=resnet_eps, resnet_act_fn=resnet_act_fn,
                                  resnet_groups=resnet_groups, cross_attention_dim=cross_attention_dim,
                                  attn_num_head_channels=attn_num_head_channels,
                                  use_linear_projection=use_linear_projection)
    raise ValueError(f"{up_block_type} does not exist.")
