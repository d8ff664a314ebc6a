"""Mirror of diffusers' `UNetSpatioTemporalConditionModel` (Stable Video Diffusion) as the reference drives it:
`MaskStableVideoDiffusionPipeline.__call__` (models/pipeline.py:223-466; loop :416-450) feeds it the 9-channel
`cat([mask, latents, image_latents], dim=2)` (:422) from train_svd.py:756-777 (BASELINE config 4).

Same constructor config, sub-module names (-> state_dict keys) and forward signature as diffusers 0.24
(`forward(sample [B, F, C, H, W], timestep, encoder_hidden_states [B, 1, D], added_time_ids [B, 3])` -> `.sample`
[B, F, 4, H, W]); executed on the same sm_90a kernels as the UNet3D path:

  SpatioTemporalResBlock      = ResnetBlock2D (implicit-GEMM convs, per-sample time-embedding bias in the epilogue)
                                + TemporalResnetBlock (GroupNorm over [b, c, f, h, w] + SiLU -> 3-tap temporal implicit GEMM,
                                twice, + identity) + AlphaBlender (`aab_axpby`)
  TransformerSpatioTemporalModel = spatial BasicTransformerBlock (flash d64 self-attention; the cross-attention has ONE key
                                -- the image embedding -- so softmax is identically 1 and the attention output is the vector
                                to_out(to_v(context)) of the sample, added with `aab_add_rowvec`)
                                + frame position embedding + TemporalBasicTransformerBlock (attention over the F frames of
                                every pixel with the gather-in-kernel temporal attention, no permutes) + AlphaBlender
Activation layout as in engine.py: [rows, C] with rows = (b, f, y, x).

Restrictions (raise, never fall back): attention head dim 64 (the SVD checkpoints: 320/5, 640/10, 1280/20), F <= 128, 16-bit
weights on a CUDA device.  Parity: tests/test_gpu_svd.py against the oracle restatement (oracle/shim/diffusers/_svd.py —
leaf semantics recalled from diffusers 0.24, unpinned; composition pinned to the verbatim reference pipeline).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple, Union

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from .layers import (Attention, BasicTransformerBlock, Downsample2D, FeedForward, ResnetBlock2D, TimestepEmbedding,
                     Upsample2D, _ParamsOnly)
from .modeling import BaseOutput, ModelBase, capture_config


# ------------------------------------------------------------------------------------------------ parameter containers
class AlphaBlender(_ParamsOnly):
    def __init__(self, alpha: float, merge_strategy: str = "learned_with_images", switch_spatial_to_temporal_mix=False):
        super().__init__()
        if merge_strategy not in ("learned", "learned_with_images"):
            raise NotImplementedError(f"merge_strategy {merge_strategy!r}")
        self.merge_strategy = merge_strategy
        self.switch_spatial_to_temporal_mix = switch_spatial_to_temporal_mix
        self.mix_factor = nn.Parameter(torch.tensor([float(alpha)]))


class TemporalResnetBlock(_ParamsOnly):
    def __init__(self, in_channels, out_channels=None, temb_channels=512, eps=1e-6):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        if out_channels != in_channels:
            raise NotImplementedError("TemporalResnetBlock with a channel change (conv_shortcut) is not used by SVD")
        self.in_channels, self.out_channels, self.eps = in_channels, out_channels, eps
        self.norm1 = nn.GroupNorm(32, in_channels, eps=eps)
        self.conv1 = nn.Conv3d(in_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))
        self.time_emb_proj = nn.Linear(temb_channels, out_channels) if temb_channels is not None else None
        self.norm2 = nn.GroupNorm(32, out_channels, eps=eps)
        self.conv2 = nn.Conv3d(out_channels, out_channels, (3, 1, 1), padding=(1, 0, 0))


class SpatioTemporalResBlock(_ParamsOnly):
    def __init__(self, in_channels, out_channels=None, temb_channels=512, eps=1e-6, temporal_eps=None, merge_factor=0.5,
                 merge_strategy="learned_with_images", switch_spatial_to_temporal_mix=False):
        super().__init__()
        out_channels = out_channels if out_channels is not None else in_channels
        self.spatial_res_block = ResnetBlock2D(in_channels=in_channels, out_channels=out_channels,
                                               temb_channels=temb_channels, eps=eps)
        self.temporal_res_block = TemporalResnetBlock(out_channels, out_channels, temb_channels=temb_channels,
                                                      eps=temporal_eps if temporal_eps is not None else eps)
        self.time_mixer = AlphaBlender(merge_factor, merge_strategy, switch_spatial_to_temporal_mix)


class _FeedForwardOut(_ParamsOnly):
    """FeedForward(dim, dim_out=...) (GEGLU): same parameter names as diffusers' FeedForward."""

    def __init__(self, dim, dim_out, mult=4):
        super().__init__()
        from .layers import GEGLU
        self.net = nn.ModuleList([GEGLU(dim, dim * mult), nn.Dropout(0.0), nn.Linear(dim * mult, dim_out)])


class TemporalBasicTransformerBlock(_ParamsOnly):
    def __init__(self, dim, time_mix_inner_dim, num_attention_heads, attention_head_dim, cross_attention_dim=None):
        super().__init__()
        if dim != time_mix_inner_dim:
            raise NotImplementedError("time_mix_inner_dim != dim is not used by SVD")
        self.norm_in = nn.LayerNorm(dim)
        self.ff_in = _FeedForwardOut(dim, time_mix_inner_dim)
        self.norm1 = nn.LayerNorm(time_mix_inner_dim)
        self.attn1 = Attention(time_mix_inner_dim, heads=num_attention_heads, dim_head=attention_head_dim)
        if cross_attention_dim is not None:
            self.norm2 = nn.LayerNorm(time_mix_inner_dim)
            self.attn2 = Attention(time_mix_inner_dim, cross_attention_dim=cross_attention_dim, heads=num_attention_heads,
                                   dim_head=attention_head_dim)
        else:
            self.norm2, self.attn2 = None, None
        self.norm3 = nn.LayerNorm(time_mix_inner_dim)
        self.ff = FeedForward(time_mix_inner_dim)


class TransformerSpatioTemporalModel(_ParamsOnly):
    def __init__(self, num_attention_heads=16, attention_head_dim=88, in_channels=320, out_channels=None, num_layers=1,
                 cross_attention_dim=None):
        super().__init__()
        if attention_head_dim != 64:
            raise ValueError("the sm_90a attention kernels are specialised for head_dim 64 (SVD: 320/5, 640/10, 1280/20)")
        inner = num_attention_heads * attention_head_dim
        if inner != in_channels:
            raise NotImplementedError("inner_dim != in_channels is not used by SVD")
        self.heads, self.head_dim, self.in_channels = num_attention_heads, attention_head_dim, in_channels
        self.norm = nn.GroupNorm(32, in_channels, eps=1e-6)
        self.proj_in = nn.Linear(in_channels, inner)
        self.transformer_blocks = nn.ModuleList([
            BasicTransformerBlock(inner, num_attention_heads, attention_head_dim, cross_attention_dim=cross_attention_dim)
            for _ in range(num_layers)])
        self.temporal_transformer_blocks = nn.ModuleList([
            TemporalBasicTransformerBlock(inner, inner, num_attention_heads, attention_head_dim,
                                          cross_attention_dim=cross_attention_dim) for _ in range(num_layers)])
        self.time_pos_embed = TimestepEmbedding(in_channels, in_channels * 4, out_dim=in_channels)
        self.time_mixer = AlphaBlender(0.5, "learned_with_images")
        self.proj_out = nn.Linear(inner, in_channels)


# ------------------------------------------------------------------------------------------------ weight preparation
def _alpha(m: AlphaBlender) -> float:
    """image_only_indicator is all zeros on this path -> alpha = sigmoid(mix_factor) for both strategies.  Kept in fp32 and
    not rounded to the model dtype (the stock 16-bit AlphaBlender rounds alpha first, then takes 1 - alpha in 16 bits):
    `aab_axpby` gets alpha and 1 - alpha as fp32 coefficients, as the fp32 reference computes them."""
    a = float(torch.sigmoid(m.mix_factor.detach().float()).item())
    return 1.0 - a if m.switch_spatial_to_temporal_mix else a


def prepare_svd_modules(prep: E.Prepared, root: nn.Module):
    dt = prep.dtype
    E.prepare_module(prep, root)                    # ResnetBlock2D, Down/Upsample2D, BasicTransformerBlock, TimestepEmbedding
    for m in root.modules():
        if id(m) in prep.m:
            continue
        if isinstance(m, TemporalResnetBlock):
            prep.put(m, {"n1": E.prep_norm(m.norm1), "c1": E.prep_conv3d_t(m.conv1, dt), "n2": E.prep_norm(m.norm2),
                         "c2": E.prep_conv3d_t(m.conv2, dt)})
        elif isinstance(m, SpatioTemporalResBlock):
            prep.put(m, {"alpha": _alpha(m.time_mixer)})
        elif isinstance(m, TemporalBasicTransformerBlock):
            a1 = m.attn1
            d = {"n_in": E.prep_norm(m.norm_in), "ffi1": E.prep_linear(m.ff_in.net[0].proj, dt),
                 "ffi2": E.prep_linear(m.ff_in.net[2], dt), "n1": E.prep_norm(m.norm1),
                 "qkv1": E._w(torch.cat([a1.to_q.weight, a1.to_k.weight, a1.to_v.weight], dim=0), dt),
                 "o1": E.prep_linear(a1.to_out[0], dt), "n3": E.prep_norm(m.norm3),
                 "ff1": E.prep_linear(m.ff.net[0].proj, dt), "ff2": E.prep_linear(m.ff.net[2], dt)}
            if m.attn2 is not None:
                d["v2"] = E._w(m.attn2.to_v.weight, dt)
                d["o2"] = E.prep_linear(m.attn2.to_out[0], dt)
            prep.put(m, d)
        elif isinstance(m, TransformerSpatioTemporalModel):
            prep.put(m, {"n": E.prep_norm(m.norm), "pi": E.prep_linear(m.proj_in, dt), "po": E.prep_linear(m.proj_out, dt),
                         "alpha": _alpha(m.time_mixer)})
    # the single-key cross-attention of the spatial blocks only needs to_v and to_out
    for m in root.modules():
        if isinstance(m, BasicTransformerBlock) and m.attn2 is not None and m.attn2.is_cross:
            d = prep.get(m)
            if "v2" not in d:
                d["v2"] = E._w(m.attn2.to_v.weight, dt)


# ------------------------------------------------------------------------------------------------ forward pieces
def _single_key_cross(p: dict, ctx_vec: torch.Tensor) -> torch.Tensor:
    """Attention with ONE key/value row per sample: softmax over one key is 1, so attn(q, k, v) = to_out(to_v(context)) for
    every query token.  ctx_vec [B, D] 16-bit -> fp32 [B, C] (bias included)."""
    v = ops.linear(ctx_vec, p["v2"])
    return ops.linear(v, p["o2"][0], p["o2"][1], out_f32=True)


def st_resblock_forward(ctx: E.Ctx, m: SpatioTemporalResBlock, x, g: E.Geo, skip=None):
    xs = E.resnet_forward(ctx, m.spatial_res_block, x, g, skip=skip)
    t = m.temporal_res_block
    p = ctx.prep.get(t)
    c = t.out_channels
    bias2 = None
    if t.time_emb_proj is not None and ctx.temb_all is not None:
        off = ctx.temb_off[id(t)]
        bias2 = ctx.temb_all[:, off: off + c]
    h = ops.groupnorm(xs, g.b, g.t * g.hw, p["n1"][0], p["n1"][1], t.eps, True, 32)
    h = ops.tconv3(h, g.b, g.t, g.hw, p["c1"][0], p["c1"][1], bias2=bias2, rows_per_bias2=g.t * g.hw)
    h = ops.groupnorm(h, g.b, g.t * g.hw, p["n2"][0], p["n2"][1], t.eps, True, 32)
    xt = ops.tconv3(h, g.b, g.t, g.hw, p["c2"][0], p["c2"][1], residual=xs)
    a = ctx.prep.get(m)["alpha"]
    return ops.axpby(xs, xt, a, 1.0 - a)


def st_transformer_forward(ctx: E.Ctx, m: TransformerSpatioTemporalModel, x, g: E.Geo):
    p = ctx.prep.get(m)
    inner = m.heads * 64
    hs = ops.groupnorm(x, g.n, g.hw, p["n"][0], p["n"][1], 1e-6, False, 32)
    hs = ops.linear(hs, p["pi"][0], p["pi"][1])
    # frame position embedding: time_pos_embed(time_proj(arange(F)))  -> fp32 [F, C]
    te = ctx.prep.get(m.time_pos_embed)
    t_emb = ops.timestep_embed(ctx.frame_idx, g.t, m.in_channels, ctx.prep.dtype)
    e1 = ops.linear(t_emb, te["l1"][0], te["l1"][1], act=ops.ACT_SILU)
    emb = ops.linear(e1, te["l2"][0], te["l2"][1], out_f32=True)
    for blk, tblk in zip(m.transformer_blocks, m.temporal_transformer_blocks):
        bp = ctx.prep.get(blk)
        n1 = ops.layernorm(hs, bp["n1"][0], bp["n1"][1])
        qkv = ops.linear(n1, bp["qkv1"])
        a = ops.flash_attn_d64(qkv, 0, qkv, inner, 2 * inner, g.n, g.hw, g.hw, m.heads)
        hs = ops.linear(a, bp["o1"][0], bp["o1"][1], residual=hs)
        if blk.attn2 is not None:
            ops.add_rowvec(hs, _single_key_cross(bp, ctx.ehs), g.t * g.hw, g.b, inplace=True)
        n3 = ops.layernorm(hs, bp["n3"][0], bp["n3"][1])
        hs = E._ff(ctx, bp, hs, n3)
        # ---- temporal block on hs + frame embedding (tokens stay in (b, f, s) order; attention gathers over f)
        tp = ctx.prep.get(tblk)
        mix = ops.add_rowvec(hs, emb, g.hw, g.t)
        h = ops.layernorm(mix, tp["n_in"][0], tp["n_in"][1])
        f = ops.linear(h, tp["ffi1"][0], tp["ffi1"][1], geglu=True)
        h = ops.linear(f, tp["ffi2"][0], tp["ffi2"][1], residual=mix)
        n = ops.layernorm(h, tp["n1"][0], tp["n1"][1])
        qkv = ops.linear(n, tp["qkv1"])
        a = ops.temporal_attn(qkv, g.b, g.t, g.hw, m.heads, 0, inner, 2 * inner)
        h = ops.linear(a, tp["o1"][0], tp["o1"][1], residual=h)
        if tblk.attn2 is not None:
            # diffusers builds `time_context` in (h*w, batch) order but the block's tokens are (batch, h*w): token (b, s)
            # reads the context of sample (b * S + s) % B (kept bug-compatible)
            ops.add_rowvec(h, _single_key_cross(tp, ctx.ehs), g.hw, g.b, mode=1, mod2=g.t, inplace=True)
        n3 = ops.layernorm(h, tp["n3"][0], tp["n3"][1])
        h = E._ff(ctx, tp, h, n3)
        al = p["alpha"]
        hs = ops.axpby(hs, h, al, 1.0 - al)
    return ops.linear(hs, p["po"][0], p["po"][1], residual=x)


# ------------------------------------------------------------------------------------------------ blocks
class _Blk(nn.Module):
    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("blocks are executed through UNetSpatioTemporalConditionModel.forward (sm_90a engine)")


class DownBlockSpatioTemporal(_Blk):
    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, add_downsample=True):
        super().__init__()
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(in_channels if i == 0 else out_channels, out_channels,
                                                             temb_channels, eps=1e-5) for i in range(num_layers)])
        self.downsamplers = (nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                         name="op")]) if add_downsample else None)

    def run(self, ctx, x, g):
        outs = []
        for r in self.resnets:
            x = st_resblock_forward(ctx, r, x, g)
            outs.append((x, g))
        if self.downsamplers is not None:
            x = E.downsample_forward(ctx, self.downsamplers[0], x, g)
            g = g.down()
            outs.append((x, g))
        return x, g, outs


class CrossAttnDownBlockSpatioTemporal(_Blk):
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, temb_channels, num_layers=1, transformer_layers_per_block=1,
                 num_attention_heads=1, cross_attention_dim=1280, add_downsample=True):
        super().__init__()
        if isinstance(transformer_layers_per_block, int):
            transformer_layers_per_block = [transformer_layers_per_block] * num_layers
        self.resnets = nn.ModuleList([SpatioTemporalResBlock(in_channels if i == 0 else out_channels, out_channels,
                                                             temb_channels, eps=1e-6) for i in range(num_layers)])
        self.attentions = nn.ModuleList([
            TransformerSpatioTemporalModel(num_attention_heads, out_channels // num_attention_heads,
                                           in_channels=out_channels, num_layers=transformer_layers_per_block[i],
                                           cross_attention_dim=cross_attention_dim) for i in range(num_layers)])
        self.downsamplers = (nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                         padding=1, name="op")]) if add_downsample else None)

    def run(self, ctx, x, g):
        outs = []
        for r, a in zip(self.resnets, self.attentions):
            x = st_resblock_forward(ctx, r, x, g)
            x = st_transformer_forward(ctx, a, x, g)
            outs.append((x, g))
        if self.downsamplers is not None:
            x = E.downsample_forward(ctx, self.downsamplers[0], x, g)
            g = g.down()
            outs.append((x, g))
        return x, g, outs


class UNetMidBlockSpatioTemporal(_Blk):
    has_cross_attention = True

    def __init__(self, in_channels, temb_channels, num_layers=1, transformer_layers_per_block=1, num_attention_heads=1,
                 cross_attention_dim=1280):
        super().__init__()
        if isinstance(transformer_layers_per_block, int):
            transformer_layers_per_block = [transformer_layers_per_block] * num_layers
        resnets = [SpatioTemporalResBlock(in_channels, in_channels, temb_channels, eps=1e-5)]
        attentions = []
        for i in range(num_layers):
            attentions.append(TransformerSpatioTemporalModel(num_attention_heads, in_channels // num_attention_heads,
                                                             in_channels=in_channels,
                                                             num_layers=transformer_layers_per_block[i],
                                                             cross_attention_dim=cross_attention_dim))
            resnets.append(SpatioTemporalResBlock(in_channels, in_channels, temb_channels, eps=1e-5))
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)

    def run(self, ctx, x, g):
        x = st_resblock_forward(ctx, self.resnets[0], x, g)
        for a, r in zip(self.attentions, self.resnets[1:]):
            x = st_transformer_forward(ctx, a, x, g)
            x = st_resblock_forward(ctx, r, x, g)
        return x


class UpBlockSpatioTemporal(_Blk):
    def __init__(self, in_channels, prev_output_channel, out_channels, temb_channels, resolution_idx=None, num_layers=1,
                 resnet_eps=1e-6, add_upsample=True):
        super().__init__()
        resnets = []
        for i in range(num_layers):
            skip = in_channels if (i == num_layers - 1) else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(SpatioTemporalResBlock(cin + skip, out_channels, temb_channels, eps=resnet_eps))
        self.resnets = nn.ModuleList(resnets)
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)

    def run(self, ctx, x, g, skips):
        for r in self.resnets:
            skip, sg = skips.pop()
            assert (sg.h, sg.w) == (g.h, g.w)
            x = st_resblock_forward(ctx, r, x, g, skip=skip)
        if self.upsamplers is not None:
            x = E.upsample_forward(ctx, self.upsamplers[0], x, g)
            g = g.up()
        return x, g


class CrossAttnUpBlockSpatioTemporal(_Blk):
    has_cross_attention = True

    def __init__(self, in_channels, out_channels, prev_output_channel, temb_channels, resolution_idx=None, num_layers=1,
                 transformer_layers_per_block=1, resnet_eps=1e-6, num_attention_heads=1, cross_attention_dim=1280,
                 add_upsample=True):
        super().__init__()
        if isinstance(transformer_layers_per_block, int):
            transformer_layers_per_block = [transformer_layers_per_block] * num_layers
        resnets, attentions = [], []
        for i in range(num_layers):
            skip = in_channels if (i == num_layers - 1) else out_channels
            cin = prev_output_channel if i == 0 else out_channels
            resnets.append(SpatioTemporalResBlock(cin + skip, out_channels, temb_channels, eps=resnet_eps))
            attentions.append(TransformerSpatioTemporalModel(num_attention_heads, out_channels // num_attention_heads,
                                                             in_channels=out_channels,
                                                             num_layers=transformer_layers_per_block[i],
                                                             cross_attention_dim=cross_attention_dim))
        self.resnets = nn.ModuleList(resnets)
        self.attentions = nn.ModuleList(attentions)
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)

    def run(self, ctx, x, g, skips):
        for r, a in zip(self.resnets, self.attentions):
            skip, sg = skips.pop()
            assert (sg.h, sg.w) == (g.h, g.w)
            x = st_resblock_forward(ctx, r, x, g, skip=skip)
            x = st_transformer_forward(ctx, a, x, g)
        if self.upsamplers is not None:
            x = E.upsample_forward(ctx, self.upsamplers[0], x, g)
            g = g.up()
        return x, g


# ------------------------------------------------------------------------------------------------ the model
class UNetSpatioTemporalConditionOutput(BaseOutput):
    pass


class UNetSpatioTemporalConditionModel(ModelBase):
    def __init__(self, sample_size: Optional[int] = None, in_channels: int = 8, out_channels: int = 4,
                 down_block_types: Tuple[str] = ("CrossAttnDownBlockSpatioTemporal", "CrossAttnDownBlockSpatioTemporal",
                                                 "CrossAttnDownBlockSpatioTemporal", "DownBlockSpatioTemporal"),
                 up_block_types: Tuple[str] = ("UpBlockSpatioTemporal", "CrossAttnUpBlockSpatioTemporal",
                                               "CrossAttnUpBlockSpatioTemporal", "CrossAttnUpBlockSpatioTemporal"),
                 block_out_channels: Tuple[int] = (320, 640, 1280, 1280), addition_time_embed_dim: int = 256,
                 projection_class_embeddings_input_dim: int = 768, layers_per_block: Union[int, Tuple[int]] = 2,
                 cross_attention_dim: Union[int, Tuple[int]] = 1024,
                 transformer_layers_per_block: Union[int, Tuple[int]] = 1,
                 num_attention_heads: Union[int, Tuple[int]] = (5, 10, 10, 20), num_frames: int = 25):
        super().__init__()
        capture_config(self, UNetSpatioTemporalConditionModel.__init__, (), dict(
            sample_size=sample_size, in_channels=in_channels, out_channels=out_channels, down_block_types=down_block_types,
            up_block_types=up_block_types, block_out_channels=block_out_channels,
            addition_time_embed_dim=addition_time_embed_dim,
            projection_class_embeddings_input_dim=projection_class_embeddings_input_dim, layers_per_block=layers_per_block,
            cross_attention_dim=cross_attention_dim, transformer_layers_per_block=transformer_layers_per_block,
            num_attention_heads=num_attention_heads, num_frames=num_frames))
        n = len(down_block_types)
        if len(up_block_types) != n:
            raise ValueError(f"Must provide the same number of `down_block_types` as `up_block_types`. "
                             f"`down_block_types`: {down_block_types}. `up_block_types`: {up_block_types}.")
        if len(block_out_channels) != n:
            raise ValueError(f"Must provide the same number of `block_out_channels` as `down_block_types`. "
                             f"`block_out_channels`: {block_out_channels}. `down_block_types`: {down_block_types}.")
        if not isinstance(num_attention_heads, int) and len(num_attention_heads) != n:
            raise ValueError(f"Must provide the same number of `num_attention_heads` as `down_block_types`. "
                             f"`num_attention_heads`: {num_attention_heads}. `down_block_types`: {down_block_types}.")
        if out_channels != 4 or in_channels > 16:
            raise ValueError("the latent path is specialised for 4 output channels and <= 16 input channels (SVD: 8 / 9)")
        if addition_time_embed_dim % 2 or (projection_class_embeddings_input_dim % addition_time_embed_dim):
            raise ValueError("projection_class_embeddings_input_dim must be a multiple of addition_time_embed_dim")
        if isinstance(num_attention_heads, int):
            num_attention_heads = (num_attention_heads,) * n
        if isinstance(cross_attention_dim, int):
            cross_attention_dim = (cross_attention_dim,) * n
        if isinstance(layers_per_block, int):
            layers_per_block = [layers_per_block] * n
        if isinstance(transformer_layers_per_block, int):
            transformer_layers_per_block = [transformer_layers_per_block] * n
        c0 = block_out_channels[0]
        self.conv_in = nn.Conv2d(in_channels, c0, kernel_size=3, padding=1)
        ted = c0 * 4
        self.time_embedding = TimestepEmbedding(c0, ted)
        self.add_embedding = TimestepEmbedding(projection_class_embeddings_input_dim, ted)
        self.down_blocks = nn.ModuleList()
        self.up_blocks = nn.ModuleList()
        out_c = c0
        for i, t in enumerate(down_block_types):
            in_c, out_c = out_c, block_out_channels[i]
            final = i == n - 1
            if t == "DownBlockSpatioTemporal":
                blk = DownBlockSpatioTemporal(in_c, out_c, ted, num_layers=layers_per_block[i], add_downsample=not final)
            elif t == "CrossAttnDownBlockSpatioTemporal":
                blk = CrossAttnDownBlockSpatioTemporal(in_c, out_c, ted, num_layers=layers_per_block[i],
                                                       transformer_layers_per_block=transformer_layers_per_block[i],
                                                       num_attention_heads=num_attention_heads[i],
                                                       cross_attention_dim=cross_attention_dim[i], add_downsample=not final)
            else:
                raise ValueError(f"{t} does not exist.")
            self.down_blocks.append(blk)
        self.mid_block = UNetMidBlockSpatioTemporal(block_out_channels[-1], ted,
                                                    transformer_layers_per_block=transformer_layers_per_block[-1],
                                                    cross_attention_dim=cross_attention_dim[-1],
                                                    num_attention_heads=num_attention_heads[-1])
        self.num_upsamplers = 0
        rev_c = list(reversed(block_out_channels))
        rev_h = list(reversed(num_attention_heads))
        rev_l = list(reversed(layers_per_block))
        rev_x = list(reversed(cross_attention_dim))
        rev_t = list(reversed(transformer_layers_per_block))
        out_c = rev_c[0]
        for i, t in enumerate(up_block_types):
            final = i == n - 1
            prev, out_c = out_c, rev_c[i]
            in_c = rev_c[min(i + 1, n - 1)]
            if not final:
                self.num_upsamplers += 1
            if t == "UpBlockSpatioTemporal":
                blk = UpBlockSpatioTemporal(in_c, prev, out_c, ted, resolution_idx=i, num_layers=rev_l[i] + 1,
                                            add_upsample=not final)
            elif t == "CrossAttnUpBlockSpatioTemporal":
                blk = CrossAttnUpBlockSpatioTemporal(in_c, out_c, prev, ted, resolution_idx=i, num_layers=rev_l[i] + 1,
                                                     transformer_layers_per_block=rev_t[i], num_attention_heads=rev_h[i],
                                                     cross_attention_dim=rev_x[i], add_upsample=not final)
            else:
                raise ValueError(f"{t} does not exist.")
            self.up_blocks.append(blk)
        self.conv_norm_out = nn.GroupNorm(num_channels=c0, num_groups=32, eps=1e-5)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(c0, out_channels, kernel_size=3, padding=1)
        self.__dict__["_aab_prepared"] = None
        self.fuse_geglu = True

    # ------------------------------------------------------------------ weights
    def _prepared(self) -> E.Prepared:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.conv_out.weight
        if prep is not None and prep.dtype == p0.dtype and prep.device == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16) or not p0.is_cuda:
            raise TypeError("UNetSpatioTemporalConditionModel must be fp16/bf16 on a CUDA device for the sm_90a path "
                            "(train_svd.py:87 loads it in fp16 on cuda); there is no fp32/CPU fallback")
        prep = self._build_prepared(p0.dtype, p0.device)
        self.__dict__["_aab_prepared"] = prep
        return prep

    def _build_prepared(self, dt, device) -> E.Prepared:
        prep = E.Prepared(dt, device)
        with torch.no_grad():
            prepare_svd_modules(prep, self)
            own = {"conv_in": E.prep_conv3x3(self.conv_in, dt, pad_cin_to=16),
                   "norm_out": E.prep_norm(self.conv_norm_out), "conv_out": E.prep_conv3x3(self.conv_out, dt)}
            ws, bs, offs, off = [], [], {}, 0
            for m in self.modules():            # spatial ResnetBlock2D and TemporalResnetBlock both take silu(emb)
                if isinstance(m, (ResnetBlock2D, TemporalResnetBlock)) and m.time_emb_proj is not None:
                    offs[id(m)] = off
                    ws.append(m.time_emb_proj.weight.detach())
                    bs.append(m.time_emb_proj.bias.detach())
                    off += m.out_channels
            own["temb_w"] = torch.cat(ws, dim=0).to(dt).contiguous()
            own["temb_b"] = torch.cat(bs, dim=0).float().contiguous()
            own["temb_off"] = offs
            prep.put(self, own)
        return prep

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timestep, encoder_hidden_states: torch.Tensor, added_time_ids: torch.Tensor,
                return_dict: bool = True, _raw: bool = False, _x16: Optional[torch.Tensor] = None, _shape=None):
        """`_x16` / `_shape` (used by the fused SVD loop, pipeline_svd.py): the channels-last, 16-channel-padded input
        [B*F, h, w, 16] already assembled by `aab_svd_in_assemble`, with `_shape` = (B, F, C, h, w); `sample` is ignored."""
        cfg = self.config
        if _x16 is not None:
            b, nf, c, h, w = _shape
        else:
            if sample.dim() != 5 or sample.shape[2] != cfg.in_channels:
                raise ValueError(f"sample must be [batch, frames, {cfg.in_channels}, height, width], got {tuple(sample.shape)}")
            b, nf, c, h, w = sample.shape
        if nf > ops.TEMPORAL_MAX_FRAMES:       # before the first launch, not halfway through the forward
            raise NotImplementedError(f"temporal attention handles up to {ops.TEMPORAL_MAX_FRAMES} frames, got {nf}")
        prep = self._prepared()
        own = prep.get(self)
        dt, dev = prep.dtype, prep.device
        if any(s % (2 ** self.num_upsamplers) for s in (h, w)):
            raise ValueError("latent height/width must be multiples of 2**num_upsamplers (diffusers' SVD UNet has no "
                             "upsample_size path either)")
        if encoder_hidden_states.dim() != 3 or encoder_hidden_states.shape[0] != b:
            raise ValueError("encoder_hidden_states must be [batch, 1, cross_attention_dim] (one image embedding per sample)")
        if encoder_hidden_states.shape[1] != 1:
            # diffusers 0.24 TransformerSpatioTemporalModel.forward broadcasts the first frame's context to
            # (h*w, batch, 1, dim) with a literal 1: a multi-token context (TextStableVideoDiffusionPipeline with
            # condition_type != "image", models/pipeline.py:579-587) fails there with exactly this error
            raise RuntimeError(f"The expanded size of the tensor (1) must match the existing size "
                               f"({encoder_hidden_states.shape[1]}) at non-singleton dimension 2.  Target sizes: "
                               f"[{h // 1 * w}, {b}, 1, {encoder_hidden_states.shape[-1]}].  Tensor sizes: "
                               f"[1, {b}, {encoder_hidden_states.shape[1]}, {encoder_hidden_states.shape[-1]}]")
        if added_time_ids.shape != (b, cfg.projection_class_embeddings_input_dim // cfg.addition_time_embed_dim):
            raise ValueError(
                f"Model expects an added time embedding vector of length {cfg.projection_class_embeddings_input_dim}, but a "
                f"vector of {added_time_ids.shape[-1] * cfg.addition_time_embed_dim} was created.")
        g = E.Geo(b, nf, h, w)
        ctx = E.Ctx(prep, g)
        ctx.fuse_geglu = self.fuse_geglu
        ctx.temb_off = own["temb_off"]
        ctx.frame_idx = torch.arange(nf, device=dev, dtype=torch.float32)
        ehs = encoder_hidden_states.to(device=dev, dtype=dt)
        ctx.ehs = ehs.reshape(b, ehs.shape[-1]).contiguous()
        # time + added-condition embedding (diffusers forward: emb = time_embedding(time_proj(t)) + add_embedding(...))
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([float(timestep)], dtype=torch.float32, device=dev)
        timestep = timestep.to(device=dev, dtype=torch.float32).reshape(-1)
        if timestep.numel() not in (1, b):
            raise ValueError(f"`timestep` has {timestep.numel()} values for a batch of {b}")
        c0 = self.conv_in.out_channels
        te, ae = prep.get(self.time_embedding), prep.get(self.add_embedding)
        t_emb = ops.timestep_embed(timestep, b, c0, dt)
        e1 = ops.linear(ops.linear(t_emb, te["l1"][0], te["l1"][1], act=ops.ACT_SILU), te["l2"][0], te["l2"][1])
        ids = added_time_ids.to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
        a_emb = ops.timestep_embed(ids, ids.numel(), cfg.addition_time_embed_dim, dt).view(b, -1)
        h2 = ops.linear(a_emb, ae["l1"][0], ae["l1"][1], act=ops.ACT_SILU)
        semb = ops.linear(h2, ae["l2"][0], ae["l2"][1], residual=e1, act=ops.ACT_SILU)     # silu(emb + aug_emb)
        ctx.temb_all = ops.linear(semb, own["temb_w"], own["temb_b"], out_f32=True)

        x16 = _x16 if _x16 is not None else ops.image_to_nhwc16(sample.to(dt).reshape(b * nf, c, h, w))
        x = ops.conv3x3(x16, own["conv_in"][0], own["conv_in"][1])
        trace = self.__dict__.get("_trace")
        if trace is not None:
            trace.append(("conv_in", x, g))
        skips = [(x, g)]
        for i, blk in enumerate(self.down_blocks):
            x, g2, outs = blk.run(ctx, x, g)
            skips.extend(outs)
            g = g2
            if trace is not None:
                trace.append((f"down_blocks.{i}", x, g))
        x = self.mid_block.run(ctx, x, g)
        if trace is not None:
            trace.append(("mid_block", x, g))
        for i, blk in enumerate(self.up_blocks):
            x, g = blk.run(ctx, x, g, skips)
            if trace is not None:
                trace.append((f"up_blocks.{i}", x, g))
        x = ops.groupnorm(x, g.n, g.hw, own["norm_out"][0], own["norm_out"][1], self.conv_norm_out.eps, True, 32)
        y = ops.conv3x3(x.view(g.n, g.h, g.w, c0), own["conv_out"][0], own["conv_out"][1], out_f32=True)
        if _raw:
            return y, g                     # fp32 [B*F*h*w, 4] channels-last
        out = ops.svd_out_finalize(y, b, nf, h, w, dt)
        if not return_dict:
            return (out,)
        return UNetSpatioTemporalConditionOutput(sample=out)
