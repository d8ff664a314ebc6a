"""Mirror of the reference's `models/layerdiffuse_VAE.py` (SURVEY row f4, the transparent-video branch):

  LatentTransparencyOffsetEncoder   :17-41   RGBA image -> latent offset, nine 3x3 convs with SiLU (called once per clip at
                                             train_transparent_i2v_stage2.py:415)
  UNet384                           :44-177  the LayerDiffuse alpha decoder: decoded RGB frames + SD latents -> RGBA,
                                             called at models/pipeline_stage2.py:308 for every generated frame

Same constructor arguments, sub-module names and `state_dict()` keys as the reference classes (which build their blocks with
diffusers 0.24 `get_down_block` / `get_up_block` / `UNetMidBlock2D`: DownBlock2D x3, AttnDownBlock2D, AttnUpBlock2D, UpBlock2D x3,
`temb_channels=None`, GroupNorm(4)), so the reference's `vae_alpha_decoder.pth` / `vae_alpha_encoder.pth` load unchanged.

Everything runs on the kernels of the denoising path — no new GEMM or attention kernel:
  * every convolution (3x3, stride 2, 1x1) on the wgmma implicit GEMM; SiLU of the encoder in the GEMM epilogue;
    32-channel tensors in front of a stride-2 conv are widened to the 64-channel K block (`aab_pad_cols`), skip concats
    are virtual except where the first source is narrower than one K block (32 channels: one strided copy);
  * GroupNorm(4)+SiLU on the GroupNorm kernels (statistics from the producing GEMM where the tile geometry allows);
  * the head-dim-8 attention (32 heads at the 1/8 level) on the head-dim-64 flash kernel with zero-padded heads: q/k/v/out
    weights are padded once at weight-prep time, zero columns add exact zeros to Q.K^T and to the output projection, the
    softmax scale stays 1/sqrt(8);
  * `latent_conv_in` (1x1, 4 -> 128) and the `sample + sample_latent` add (:152-153) are one GEMM with a residual epilogue;
  * the pipeline's RGBA post-processing (models/pipeline_stage2.py:311-324) is fused into the decoder tail
    (`decode_rgba_u8`).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import engine as E
from . import ops
from ._lib import ACT_NONE, ACT_SILU
from .layers import Attention, Downsample2D, ResnetBlock2D, Upsample2D
from .modeling import ModelBase, capture_config


def zero_module(module):
    for p in module.parameters():
        p.detach().zero_()
    return module


def _cpad(c: int) -> int:
    return (c + 63) // 64 * 64


# ------------------------------------------------------------------------------------------------ encoder
class LatentTransparencyOffsetEncoder(ModelBase):
    """models/layerdiffuse_VAE.py:17-41.  `blocks` is the same nn.Sequential (conv at even indices, SiLU at odd ones), so
    the checkpoint keys are `blocks.{0,2,...,16}.{weight,bias}`."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        capture_config(self, LatentTransparencyOffsetEncoder.__init__, (), {})
        spec = [(4, 32, 1), (32, 32, 1), (32, 64, 2), (64, 64, 1), (64, 128, 2), (128, 128, 1), (128, 256, 2), (256, 256, 1)]
        mods = []
        for ci, co, st in spec:
            mods += [nn.Conv2d(ci, co, kernel_size=3, padding=1, stride=st), nn.SiLU()]
        mods.append(zero_module(nn.Conv2d(256, 4, kernel_size=3, padding=1, stride=1)))
        self.blocks = nn.Sequential(*mods)
        self.__dict__["_aab_prepared"] = None

    def _convs(self):
        return [m for m in self.blocks if isinstance(m, nn.Conv2d)]

    def _prepared(self) -> E.Prepared:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.blocks[0].weight
        if prep is not None and prep.dtype == p0.dtype and prep.device == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16) or not p0.is_cuda:
            raise TypeError("LatentTransparencyOffsetEncoder must be fp16/bf16 on a CUDA device for the sm_90a path (no fallback)")
        prep = self._build_prepared(p0.dtype, p0.device)
        self.__dict__["_aab_prepared"] = prep
        return prep

    def _build_prepared(self, dt, device) -> E.Prepared:
        prep = E.Prepared(dt, device)
        with torch.no_grad():
            convs = self._convs()
            ws = []
            for i, c in enumerate(convs):
                pad = 8 if i == 0 else (_cpad(c.in_channels) if c.stride[0] == 2 else None)
                ws.append(E.prep_conv3x3(c, dt, pad_cin_to=pad))
            prep.put(self, {"convs": ws})
        return prep

    @torch.no_grad()
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x [b, 4, H, W] (RGB in [-1, 1], alpha in [0, 1]; H, W multiples of 8) -> [b, 4, H/8, W/8] in x.dtype."""
        prep = self._prepared()
        n, c, hh, ww = x.shape
        if c != 4 or hh % 8 or ww % 8:
            raise ValueError("LatentTransparencyOffsetEncoder expects [b, 4, H, W] with H, W multiples of 8")
        ws = prep.get(self)["convs"]
        convs = self._convs()
        h = ops.image_to_nhwc8(x.to(prep.dtype))                      # [n, H, W, 8]
        for i, (conv, (w, b)) in enumerate(zip(convs, ws)):
            last = i == len(convs) - 1
            act = ACT_NONE if last else ACT_SILU
            if conv.stride[0] == 2:
                if h.shape[-1] % 64:
                    h = ops.pad_cols(h.view(-1, h.shape[-1]), _cpad(h.shape[-1])).view(n, hh, ww, -1)
                y = ops.conv3x3_stride2(h, w, b, pad_mode="sym", act=act)
                hh, ww = hh // 2, ww // 2
            else:
                y = ops.conv3x3(h, w, b, act=act, out_f32=last)
            h = y.view(n, hh, ww, -1) if not last else y
        return ops.svd_out_finalize(h, 1, n, hh, ww, prep.dtype)[0]   # [n, 4, h, w]

    def __call__(self, x):
        return self.forward(x)


# ------------------------------------------------------------------------------------------------ decoder blocks (containers)
def _resnet(cin, cout, groups, eps, scale=1.0):
    return ResnetBlock2D(in_channels=cin, out_channels=cout, temb_channels=None, groups=groups, eps=eps,
                         output_scale_factor=scale)


def _attention(ch, head_dim, groups, eps, scale=1.0):
    return Attention(ch, heads=ch // head_dim, dim_head=head_dim, bias=True, norm_num_groups=groups, eps=eps,
                     residual_connection=True, rescale_output_factor=scale)


class DownBlock2D(nn.Module):
    def __init__(self, in_channels, out_channels, num_layers, add_downsample, groups, eps, downsample_padding=1):
        super().__init__()
        self.resnets = nn.ModuleList([_resnet(in_channels if i == 0 else out_channels, out_channels, groups, eps)
                                      for i in range(num_layers)])
        self.downsamplers = (nn.ModuleList([Downsample2D(out_channels, use_conv=True, out_channels=out_channels,
                                                         padding=downsample_padding, name="op")]) if add_downsample else None)


class AttnDownBlock2D(DownBlock2D):
    def __init__(self, in_channels, out_channels, num_layers, add_downsample, groups, eps, attention_head_dim,
                 downsample_padding=1):
        super().__init__(in_channels, out_channels, num_layers, add_downsample, groups, eps, downsample_padding)
        self.attentions = nn.ModuleList([_attention(out_channels, attention_head_dim, groups, eps) for _ in range(num_layers)])


class UNetMidBlock2D(nn.Module):
    def __init__(self, channels, groups, eps, attention_head_dim, output_scale_factor=1.0):
        super().__init__()
        self.attentions = nn.ModuleList([_attention(channels, attention_head_dim, groups, eps, output_scale_factor)])
        self.resnets = nn.ModuleList([_resnet(channels, channels, groups, eps, output_scale_factor) for _ in range(2)])


class UpBlock2D(nn.Module):
    def __init__(self, in_channels, prev_output_channel, out_channels, num_layers, add_upsample, groups, eps):
        super().__init__()
        res = []
        for i in range(num_layers):
            skip_c = in_channels if i == num_layers - 1 else out_channels
            in_c = prev_output_channel if i == 0 else out_channels
            res.append(_resnet(in_c + skip_c, out_channels, groups, eps))
        self.resnets = nn.ModuleList(res)
        self.upsamplers = (nn.ModuleList([Upsample2D(out_channels, use_conv=True, out_channels=out_channels)])
                           if add_upsample else None)


class AttnUpBlock2D(UpBlock2D):
    def __init__(self, in_channels, prev_output_channel, out_channels, num_layers, add_upsample, groups, eps,
                 attention_head_dim):
        super().__init__(in_channels, prev_output_channel, out_channels, num_layers, add_upsample, groups, eps)
        self.attentions = nn.ModuleList([_attention(out_channels, attention_head_dim, groups, eps) for _ in range(num_layers)])


_DOWN = {"DownBlock2D": DownBlock2D, "AttnDownBlock2D": AttnDownBlock2D}
_UP = {"UpBlock2D": UpBlock2D, "AttnUpBlock2D": AttnUpBlock2D}


# ------------------------------------------------------------------------------------------------ UNet384
class UNet384(ModelBase):
    def __init__(self, in_channels: int = 3, out_channels: int = 4,
                 down_block_types: Tuple[str] = ("DownBlock2D", "DownBlock2D", "DownBlock2D", "AttnDownBlock2D"),
                 up_block_types: Tuple[str] = ("AttnUpBlock2D", "UpBlock2D", "UpBlock2D", "UpBlock2D"),
                 block_out_channels: Tuple[int] = (32, 64, 128, 256), layers_per_block: int = 2,
                 mid_block_scale_factor: float = 1, downsample_padding: int = 1, downsample_type: str = "conv",
                 upsample_type: str = "conv", dropout: float = 0.0, act_fn: str = "silu",
                 attention_head_dim: Optional[int] = 8, norm_num_groups: int = 4, norm_eps: float = 1e-5):
        super().__init__()
        capture_config(self, UNet384.__init__, (), dict(
            in_channels=in_channels, out_channels=out_channels, down_block_types=down_block_types,
            up_block_types=up_block_types, block_out_channels=block_out_channels, layers_per_block=layers_per_block,
            mid_block_scale_factor=mid_block_scale_factor, downsample_padding=downsample_padding,
            downsample_type=downsample_type, upsample_type=upsample_type, dropout=dropout, act_fn=act_fn,
            attention_head_dim=attention_head_dim, norm_num_groups=norm_num_groups, norm_eps=norm_eps))
        if in_channels > 8 or out_channels != 4:
            raise ValueError("UNet384 mirror: at most 8 image channels in, 4 (RGBA) out")
        if len(block_out_channels) != 4 or len(down_block_types) != 4 or len(up_block_types) != 4:
            raise ValueError("UNet384.forward adds the latent before down block 3 and asserts 4 down blocks "
                             "(models/layerdiffuse_VAE.py:152,158)")
        if act_fn not in ("silu", "swish") or downsample_type != "conv" or upsample_type != "conv" or downsample_padding != 1:
            raise NotImplementedError("UNet384 mirror supports the reference's defaults: silu, conv resampling, padding 1")
        if any(c % 8 or c % norm_num_groups for c in block_out_channels):
            raise ValueError("block_out_channels must be multiples of 8 and of norm_num_groups")
        for t in tuple(down_block_types) + tuple(up_block_types):
            if t not in _DOWN and t not in _UP:
                raise ValueError(f"{t} does not exist.")
        ch, g, e = list(block_out_channels), norm_num_groups, norm_eps
        self.conv_in = nn.Conv2d(in_channels, ch[0], kernel_size=3, padding=(1, 1))
        self.latent_conv_in = zero_module(nn.Conv2d(4, ch[2], kernel_size=1))
        self.down_blocks = nn.ModuleList([])
        self.mid_block = None
        self.up_blocks = nn.ModuleList([])
        out_c = ch[0]
        for i, t in enumerate(down_block_types):
            in_c, out_c = out_c, ch[i]
            final = i == len(ch) - 1
            hd = attention_head_dim if attention_head_dim is not None else out_c
            if t == "AttnDownBlock2D":
                if out_c % hd or hd > 64:
                    raise ValueError("attention_head_dim must divide the channel count and be <= 64")
                self.down_blocks.append(AttnDownBlock2D(in_c, out_c, layers_per_block, not final, g, e, hd))
            else:
                self.down_blocks.append(DownBlock2D(in_c, out_c, layers_per_block, not final, g, e))
        hd = attention_head_dim if attention_head_dim is not None else ch[-1]
        if ch[-1] % hd or hd > 64:
            raise ValueError("attention_head_dim must divide the channel count and be <= 64")
        self.mid_block = UNetMidBlock2D(ch[-1], g, e, hd, mid_block_scale_factor)
        rev = list(reversed(ch))
        out_c = rev[0]
        for i, t in enumerate(up_block_types):
            prev, out_c = out_c, rev[i]
            in_c = rev[min(i + 1, len(ch) - 1)]
            final = i == len(ch) - 1
            hd = attention_head_dim if attention_head_dim is not None else out_c
            if t == "AttnUpBlock2D":
                if out_c % hd or hd > 64:
                    raise ValueError("attention_head_dim must divide the channel count and be <= 64")
                self.up_blocks.append(AttnUpBlock2D(in_c, prev, out_c, layers_per_block + 1, not final, g, e, hd))
            else:
                self.up_blocks.append(UpBlock2D(in_c, prev, out_c, layers_per_block + 1, not final, g, e))
        self.conv_norm_out = nn.GroupNorm(num_channels=ch[0], num_groups=g, eps=e)
        self.conv_act = nn.SiLU()
        self.conv_out = nn.Conv2d(ch[0], out_channels, kernel_size=3, padding=1)
        self.frame_chunk = 16
        self.__dict__["_aab_prepared"] = None

    # ------------------------------------------------------------------ weights
    def _prepared(self) -> E.Prepared:
        prep = self.__dict__.get("_aab_prepared")
        p0 = self.conv_in.weight
        if prep is not None and prep.dtype == p0.dtype and prep.device == p0.device:
            return prep
        if p0.dtype not in (torch.float16, torch.bfloat16) or not p0.is_cuda:
            raise TypeError("UNet384 must be fp16/bf16 on a CUDA device for the sm_90a path (no fallback)")
        prep = self._build_prepared(p0.dtype, p0.device)
        self.__dict__["_aab_prepared"] = prep
        return prep

    @staticmethod
    def _prep_attention(m: Attention, dt):
        """q/k/v/out weights with every head zero-padded from dim_head to 64 columns (the flash kernel's head width)."""
        c, hds, d = m.to_q.in_features, m.heads, m.dim_head

        def pad_rows(lin):
            w = lin.weight.detach().float().view(hds, d, c)
            wp = torch.zeros((hds, 64, c), dtype=torch.float32, device=w.device)
            wp[:, :d] = w
            bp = torch.zeros((hds, 64), dtype=torch.float32, device=w.device)
            bp[:, :d] = lin.bias.detach().float().view(hds, d)
            return wp.view(hds * 64, c), bp.view(-1)
        ws, bs = zip(*(pad_rows(l) for l in (m.to_q, m.to_k, m.to_v)))
        wo = m.to_out[0].weight.detach().float().view(-1, hds, d)
        wop = torch.zeros((wo.shape[0], hds, 64), dtype=torch.float32, device=wo.device)
        wop[:, :, :d] = wo
        return {"gn": E.prep_norm(m.group_norm), "qkv": torch.cat(ws, dim=0).to(dt).contiguous(),
                "qkv_b": torch.cat(bs, dim=0).contiguous(), "o": (wop.view(wo.shape[0], hds * 64).to(dt).contiguous(),
                                                                 m.to_out[0].bias.detach().float().contiguous())}

    def _build_prepared(self, dt, device) -> E.Prepared:
        prep = E.Prepared(dt, device)
        with torch.no_grad():
            for m in self.modules():
                if isinstance(m, Attention):
                    prep.put(m, self._prep_attention(m, dt))
                elif isinstance(m, Downsample2D) and m.channels % 64:
                    prep.put(m, {"c": E.prep_conv3x3(m.conv, dt, pad_cin_to=_cpad(m.channels))})
            E.prepare_module(prep, self)
            wl = torch.zeros((self.latent_conv_in.out_channels, 8), dtype=torch.float32, device=self.latent_conv_in.weight.device)
            wl[:, :4] = self.latent_conv_in.weight.detach().float().reshape(-1, 4)
            prep.put(self, {"in": E.prep_conv3x3(self.conv_in, dt, pad_cin_to=8),
                            "lat": (wl.to(dt).contiguous(), self.latent_conv_in.bias.detach().float().contiguous()),
                            "norm": E.prep_norm(self.conv_norm_out),
                            "out": E.prep_conv3x3(self.conv_out, dt)})
        return prep

    # ------------------------------------------------------------------ engine pieces
    @staticmethod
    def _resnet(ctx, r, x, g, skip=None):
        if skip is not None and x.shape[1] % 64:
            x, skip = ops.cat_cols(x, skip), None          # first source narrower than a K block: one strided copy
        return E.resnet_forward(ctx, r, x, g, skip)

    @staticmethod
    def _attn(ctx, m: Attention, x, g):
        """diffusers Attention (deprecated attn-block form, AttnProcessor2_0): GroupNorm -> q,k,v (bias) ->
        softmax(Q K^T / sqrt(dim_head)) V per head -> to_out -> (+ residual) / rescale_output_factor."""
        p = ctx.prep.get(m)
        inner = m.heads * 64
        hn = ops.groupnorm(x, g.n, g.hw, p["gn"][0], p["gn"][1], m.group_norm.eps, False, m.group_norm.num_groups)
        qkv = ops.linear(hn, p["qkv"], p["qkv_b"])
        a = ops.flash_attn_d64(qkv, 0, qkv, inner, 2 * inner, g.n, g.hw, g.hw, m.heads, scale=float(m.dim_head) ** -0.5)
        return ops.linear(a, p["o"][0], p["o"][1], residual=x, out_scale=1.0 / m.rescale_output_factor, stats=True)

    @staticmethod
    def _down(ctx, ds: Downsample2D, x, g):
        p = ctx.prep.get(ds)
        c = ds.channels
        if c % 64:
            x = ops.pad_cols(x, _cpad(c))
        return ops.conv3x3_stride2(x.view(g.n, g.h, g.w, x.shape[1]), p["c"][0], p["c"][1], pad_mode="sym", stats=True)

    def _forward_chunk(self, prep, x8: torch.Tensor, lat8: torch.Tensor) -> torch.Tensor:
        """x8 [n, H, W, 8], lat8 [n, H/8, W/8, 8] channels-last 16-bit -> conv_out result [n*H*W, 4] fp32."""
        own = prep.get(self)
        n, hh, ww, _ = x8.shape
        g = E.Geo(n, 1, hh, ww)
        ctx = E.Ctx(prep, g)
        sample = ops.conv3x3(x8, own["in"][0], own["in"][1], stats=True)
        skips = [(sample, g)]
        for i, blk in enumerate(self.down_blocks):
            if i == 3:
                # sample + latent_conv_in(latent) (:146,:152-153): the 1x1 conv with the running sample as its residual
                sample = ops.linear(lat8.view(-1, 8), own["lat"][0], own["lat"][1], residual=sample, stats=True)
            attns = getattr(blk, "attentions", None)
            for j, r in enumerate(blk.resnets):
                sample = self._resnet(ctx, r, sample, g)
                if attns is not None:
                    sample = self._attn(ctx, attns[j], sample, g)
                skips.append((sample, g))
            if blk.downsamplers is not None:
                sample = self._down(ctx, blk.downsamplers[0], sample, g)
                g = E.Geo(n, 1, g.h // 2, g.w // 2)
                skips.append((sample, g))
        mid = self.mid_block
        sample = self._resnet(ctx, mid.resnets[0], sample, g)
        sample = self._attn(ctx, mid.attentions[0], sample, g)
        sample = self._resnet(ctx, mid.resnets[1], sample, g)
        for blk in self.up_blocks:
            attns = getattr(blk, "attentions", None)
            for j, r in enumerate(blk.resnets):
                skip, sg = skips.pop()
                assert (sg.h, sg.w) == (g.h, g.w)
                sample = self._resnet(ctx, r, sample, g, skip)
                if attns is not None:
                    sample = self._attn(ctx, attns[j], sample, g)
            if blk.upsamplers is not None:
                sample = E.upsample_forward(ctx, blk.upsamplers[0], sample, g)
                g = g.up()
        c0 = self.conv_out.in_channels
        h = ops.groupnorm(sample, g.n, g.hw, own["norm"][0], own["norm"][1], self.conv_norm_out.eps, True,
                          self.conv_norm_out.num_groups)
        return ops.conv3x3(h.view(g.n, g.h, g.w, c0), own["out"][0], own["out"][1], out_f32=True)

    def _check(self, hh, ww, lh, lw):
        if hh % 8 or ww % 8 or (lh, lw) != (hh // 8, ww // 8):
            raise ValueError(f"UNet384: image {hh}x{ww} must be a multiple of 8 and the latent {lh}x{lw} one eighth of it "
                             "(the reference's skip concatenation / latent add fail otherwise)")

    # ------------------------------------------------------------------ public API
    @torch.no_grad()
    def forward(self, x: torch.Tensor, latent: torch.Tensor) -> torch.Tensor:
        """models/layerdiffuse_VAE.py:145-174: x [n, 3, H, W] decoded frames, latent [n, 4, H/8, W/8] -> RGBA [n, 4, H, W]."""
        prep = self._prepared()
        n, _, hh, ww = x.shape
        self._check(hh, ww, latent.shape[-2], latent.shape[-1])
        outs = []
        for i in range(0, n, self.frame_chunk):
            xs, ls = x[i: i + self.frame_chunk].to(prep.dtype), latent[i: i + self.frame_chunk].to(prep.dtype)
            y = self._forward_chunk(prep, ops.image_to_nhwc8(xs), ops.image_to_nhwc8(ls))
            outs.append(ops.svd_out_finalize(y, 1, xs.shape[0], hh, ww, prep.dtype)[0])
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)

    def __call__(self, x, latent):
        return self.forward(x, latent)

    @torch.no_grad()
    def decode_rgba_u8(self, video: torch.Tensor, latents: torch.Tensor) -> torch.Tensor:
        """The tail of MaskedLatentToVideoPipeline.__call__ (models/pipeline_stage2.py:303-324) for batch element 0:
        `video` fp32 [b, 3, f, H, W] (decode_latents output), `latents` [b, 4, f, h, w] -> uint8 RGBA frames [f, H, W, 4]
        on the device.  The layout changes (:305-306,:310), the decoder and the alpha threshold / foreground scaling run
        without materialising the intermediate tensors."""
        prep = self._prepared()
        b, _, f, hh, ww = video.shape
        self._check(hh, ww, latents.shape[-2], latents.shape[-1])
        latents = latents.to(prep.dtype)
        outs = []
        for i in range(0, f, self.frame_chunk):
            v = video[:1, :, i: i + self.frame_chunk]
            l5 = latents[:1, :, i: i + self.frame_chunk]
            nf = v.shape[2]
            x8 = ops.video_f32_to_nhwc8(v, prep.dtype)
            lat8 = ops.image_to_nhwc8(l5[0].permute(1, 0, 2, 3))          # strided view [f, 4, h, w]; the kernel takes strides
            y = self._forward_chunk(prep, x8, lat8)
            outs.append(ops.rgba_finalize_u8(y, nf * hh * ww, prep.dtype == torch.bfloat16).view(nf, hh, ww, 4))
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=0)
